// ssq_dev3.cuh — the paired-end bookkeeping and the text stage of `bwa mem | samblaster` as SSQ_HD routines, so that the whole
// path from reads to the three SAM streams stays in HBM (ssq_pipe.cu) and tests/hostsim can run the very same routines on the CPU.
//   pestat_pair          one pair's contribution to the insert-size histogram            (upstream mem_pestat, first loop)
//   mark_primary_d       primary / secondary marking, sub, sub_n                         (upstream mem_mark_primary_se)
//   approx_mapq_d        single-end MAPQ                                                 (upstream mem_approx_mapq_se)
//   mem_pair_d           best proper pair, sub-optimal score and count                   (upstream mem_pair)
//   plan_pair / plan_single  which hits are written, with which flag and MAPQ; which need a CIGAR (lines, XA entries, mate
//                        headers)                                                        (upstream mem_sam_pe, mem_reg2sam, mem_gen_alt)
//   sam_line             one SAM record, byte for byte                                   (upstream mem_aln2sam)
//   sb_*                 samblaster on structured records: signature, discordant and splitter predicates, MC/MQ tags
//                        (upstream samblaster.cpp markDupsDiscordants / markSplitterUnmappedClipped; SURVEY §8a a16-a19)
// Reference call sites: `$BWA mem ... | $SAMBLASTER ...` at speedseq/bin/speedseq:438-439,468-469.
//
// Floating point: every double expression below is evaluated as separate IEEE operations (the translation units that include
// this header are compiled with -fmad=false; the host build has no FMA contraction either), and every transcendental comes from
// a table computed on the host with the same libm calls the reference makes (log over integers, .721*log(2*erfc(|z|/sqrt2))*a
// over the integer insert sizes of the batch) — results are bit-identical to the host evaluation by construction.
#pragma once
#include <math.h>
#include "ssq_dev2.cuh"

#define CIG_CAP 64
#define MD_CAP 512

SSQ_HD u64 hash64_d(u64 key)
{
	key += ~(key << 32); key ^= (key >> 22); key += ~(key << 13); key ^= (key >> 8);
	key += (key << 3); key ^= (key >> 15); key += ~(key << 27); key ^= (key >> 31);
	return key;
}

// host-computed tables (see the header comment)
struct MathTabs {
	const double *logn; i32 n_logn;     // log(i), i < n_logn
	const i32 *lg4343; i32 n_lg;        // (int)(4.343 * log(i + 1) + .499), i < n_lg
	const double *pen[4]; i32 pen_low[4], pen_n[4]; // per orientation: .721 * log(2 * erfc(|dist - avg| / std / sqrt2)) * a for dist = pen_low + k
};
SSQ_HD double tab_logn(const MathTabs &T, int l) { return l >= 0 && l < T.n_logn ? T.logn[l] : log((double)l); }
SSQ_HD int tab_lg4343(const MathTabs &T, int x) { return x >= 0 && x < T.n_lg ? T.lg4343[x] : (int)(4.343 * log((double)(x + 1)) + .499); }

// ---- insert-size statistics: one pair's vote (the histogram is reduced on the host, which replays the reference's sums) ----
SSQ_HD int cal_sub_d(const ssq_opts_t &o, const AlnReg *r, int n)
{
	int j;
	for (j = 1; j < n; ++j) {
		const int b_max = r[j].qb > r[0].qb ? r[j].qb : r[0].qb, e_min = r[j].qe < r[0].qe ? r[j].qe : r[0].qe;
		if (e_min > b_max) {
			const int min_l = r[j].qe - r[j].qb < r[0].qe - r[0].qb ? r[j].qe - r[j].qb : r[0].qe - r[0].qb;
			if (e_min - b_max >= min_l * o.mask_level) break;
		}
	}
	return j < n ? r[j].score : o.min_seed_len * o.a;
}
SSQ_HD bool pestat_pair(const ssq_opts_t &o, i64 l_pac, const AlnReg *r0, int n0, const AlnReg *r1, int n1, int *dir, i64 *is)
{
	if (n0 == 0 || n1 == 0) return false;
	if (cal_sub_d(o, r0, n0) > 0.8 * r0[0].score) return false;
	if (cal_sub_d(o, r1, n1) > 0.8 * r1[0].score) return false;
	if (r0[0].rid != r1[0].rid) return false;
	*dir = infer_dir(l_pac, r0[0].rb, r1[0].rb, is);
	return *is && *is <= o.max_ins;
}

// ---- primary marking ----
SSQ_HD int mark_primary_d(const ssq_opts_t &o, int n, AlnReg *a, i64 id, i32 *idx = 0)
{
	if (n == 0) return 0;
	for (int i = 0; i < n; ++i) { a[i].sub = 0; a[i].secondary = a[i].secondary_all = -1; a[i].hash = hash64_d((u64)(id + i)); }
	// (score desc, hash asc) is a total order (hash64 is a bijection), so any sort gives the reference's permutation
	if (n <= 12) ks_isort(a, 0, n, ArsHashLt()); else sort_regs(n, a, idx, ArsHashLt());
	int tmp = o.a + o.b;
	tmp = o.o_del + o.e_del > tmp ? o.o_del + o.e_del : tmp;
	tmp = o.o_ins + o.e_ins > tmp ? o.o_ins + o.e_ins : tmp;
	for (int i = 1; i < n; ++i) { // the reference's list z of non-secondary hits = the earlier hits with secondary < 0, in index order
		int j;
		for (j = 0; j < i; ++j) {
			if (a[j].secondary >= 0) continue;
			const int b_max = a[j].qb > a[i].qb ? a[j].qb : a[i].qb, e_min = a[j].qe < a[i].qe ? a[j].qe : a[i].qe;
			if (e_min > b_max) {
				const int min_l = a[i].qe - a[i].qb < a[j].qe - a[j].qb ? a[i].qe - a[i].qb : a[j].qe - a[j].qb;
				if (e_min - b_max >= min_l * o.mask_level) {
					if (a[j].sub == 0) a[j].sub = a[i].score;
					if (a[j].score - a[i].score <= tmp) ++a[j].sub_n;
					break;
				}
			}
		}
		if (j < i) a[i].secondary = j;
	}
	for (int i = 0; i < n; ++i) a[i].secondary_all = a[i].secondary;
	return n;
}

SSQ_HD int approx_mapq_d(const ssq_opts_t &o, const AlnReg &a, const MathTabs &T)
{
	int mapq, l, sub = a.sub ? a.sub : o.min_seed_len * o.a;
	sub = a.csub > sub ? a.csub : sub;
	if (sub >= a.score) return 0;
	l = a.qe - a.qb > a.re - a.rb ? a.qe - a.qb : (int)(a.re - a.rb);
	const double identity = 1. - (double)(l * o.a - a.score) / (o.a + o.b) / l;
	if (a.score == 0) mapq = 0;
	else {
		double t = l < o.mapQ_coef_len ? 1. : o.mapQ_coef_fac / tab_logn(T, l);
		t *= identity * identity;
		mapq = (int)(6.02 * (a.score - sub) / o.a * t * t + .499);
	}
	if (a.sub_n > 0) mapq -= tab_lg4343(T, a.sub_n);
	if (mapq > 60) mapq = 60;
	if (mapq < 0) mapq = 0;
	return (int)(mapq * (1. - a.frac_rep) + .499);
}
#define RAW_MAPQ(diff, a) ((int)(6.02 * (diff) / (a) + .499))

// ---- pairing ----
struct P64 { u64 x, y; };
struct P64Lt { SSQ_HD bool operator()(const P64 &a, const P64 &b) const { return a.x < b.x || (a.x == b.x && a.y < b.y); } };

// v: scratch for n[0]+n[1] entries.  The reference collects every candidate pair in a vector u, sorts it and reads the best, the
// second best and the number of near-second-best entries; here u is never stored: one sweep keeps the two largest (x,y), a
// second sweep counts (the keys (x,y) are unique, so "all but the best" is well defined).
SSQ_HD int mem_pair_d(const ssq_opts_t &o, const DevIndex &ix, const MathTabs &T, const PeStat *pes, AlnReg *const a[2], const int n[2], i64 id, int *sub, int *n_sub, int z[2], P64 *v)
{
	const i64 l_pac = ix.l_pac;
	int nv = 0;
	for (int r = 0; r < 2; ++r)
		for (int i = 0; i < n[r]; ++i) {
			const AlnReg &e = a[r][i];
			P64 key;
			key.x = e.rb < l_pac ? e.rb : (l_pac << 1) - 1 - e.rb;
			key.x = (u64)e.rid << 32 | (key.x - ix.ann_off[e.rid]);
			key.y = (u64)e.score << 32 | i << 2 | (e.rb >= l_pac) << 1 | r;
			v[nv++] = key;
		}
	if (nv <= 12) ks_isort(v, 0, nv, P64Lt()); else ks_introsort((long)nv, v, P64Lt()); // keys are unique: any sort
	P64 best, second; best.x = best.y = second.x = second.y = 0;
	u64 n_u = 0;
	int tmp = o.a + o.b;
	tmp = tmp > o.o_del + o.e_del ? tmp : o.o_del + o.e_del;
	tmp = tmp > o.o_ins + o.e_ins ? tmp : o.o_ins + o.e_ins;
	for (int pass = 0; pass < 2; ++pass) {
		int y[4] = {-1, -1, -1, -1};
		const int sub_q = (int)(second.x >> 32);
		if (pass == 1) { *n_sub = 0; if (n_u < 2) break; }
		for (int i = 0; i < nv; ++i) {
			for (int r = 0; r < 2; ++r) {
				const int dir = r << 1 | (int)(v[i].y >> 1 & 1);
				if (pes[dir].failed) continue;
				const int which = r << 1 | (int)((v[i].y & 1) ^ 1);
				if (y[which] < 0) continue;
				for (int k = y[which]; k >= 0; --k) {
					if ((int)(v[k].y & 3) != which) continue;
					const i64 dist = (i64)v[i].x - (i64)v[k].x;
					if (dist > pes[dir].high) break;
					if (dist < pes[dir].low) continue;
					double pen;
					const i64 tk = dist - T.pen_low[dir];
					if (tk >= 0 && tk < T.pen_n[dir]) pen = T.pen[dir][tk];
					else { const double ns = (dist - pes[dir].avg) / pes[dir].std; pen = .721 * log(2. * erfc(fabs(ns) * 0.70710678118654752440)) * o.a; }
					int q = (int)((v[i].y >> 32) + (v[k].y >> 32) + pen + .499);
					if (q < 0) q = 0;
					P64 p;
					p.y = (u64)k << 32 | (u32)i;
					p.x = (u64)q << 32 | (hash64_d(p.y ^ (u64)id << 8) & 0xffffffffU);
					if (pass == 0) {
						++n_u;
						if (n_u == 1 || P64Lt()(best, p)) { second = best; best = p; }
						else if (n_u == 2 || P64Lt()(second, p)) second = p;
					} else if (!(p.x == best.x && p.y == best.y) && sub_q - q <= tmp) ++*n_sub;
				}
			}
			y[v[i].y & 3] = i;
		}
	}
	if (n_u == 0) { *sub = 0; *n_sub = 0; return 0; }
	const int i = (int)(best.y >> 32), k = (int)(best.y << 32 >> 32);
	z[v[i].y & 1] = (int)(v[i].y << 32 >> 34);
	z[v[k].y & 1] = (int)(v[k].y << 32 >> 34);
	*sub = n_u > 1 ? (int)(second.x >> 32) : 0;
	return (int)(best.x >> 32);
}

// ---- what is written for a read ----
// kinds: 0 = output line (`line` = its index among the read's lines), 1 = XA entry of the line built from region xa_owner,
// 2 = mate header (the best hit of an end that is written through plan_reg2sam: position and CIGAR its mate's lines refer to)
struct PTask { i32 read, reg_idx, xa_owner; uint8_t kind, line, mapq, pad; i32 flag; };
struct ReadMeta { u32 n_tasks, n_lines; i32 extra_flag; uint8_t mode /* 0 paired lines, 1 reg2sam lines */, has_hdr, pad[2]; };

struct TaskSink { PTask *t; int n, cap, lines; bool ovf; };
SSQ_HD void add_task(TaskSink &s, int read, int reg_idx, int kind, int line, int xa_owner, int mapq, int flag)
{
	if (s.n >= s.cap) { s.ovf = true; return; }
	PTask &t = s.t[s.n++];
	t.read = read; t.reg_idx = reg_idx; t.xa_owner = xa_owner; t.kind = (uint8_t)kind; t.line = (uint8_t)line; t.mapq = (uint8_t)mapq; t.pad = 0; t.flag = flag;
}
// mem_gen_alt: secondary hits within XA_drop_ratio of their primary, at most max_XA_hits per primary.  cnt: n scratch ints
SSQ_HD void plan_xa(const ssq_opts_t &o, TaskSink &s, int read, const AlnReg *a, int n, i32 *cnt)
{
	bool any = false;
	for (int i = 0; i < n; ++i) cnt[i] = 0;
	for (int i = 0; i < n; ++i) { const int k = a[i].secondary_all; if (k >= 0 && a[i].score >= a[k].score * (double)o.XA_drop_ratio) { ++cnt[k]; any = true; } }
	if (!any) return;
	for (int i = 0; i < n; ++i) {
		const int k = a[i].secondary_all;
		if (!(k >= 0 && a[i].score >= a[k].score * (double)o.XA_drop_ratio)) continue;
		if (cnt[k] > o.max_XA_hits) continue;
		add_task(s, read, i, 1, 0, k, 0, 0);
	}
}
// mem_reg2sam without -a: every non-secondary hit above T; the first is the primary line, the others supplementary
SSQ_HD void plan_reg2sam(const ssq_opts_t &o, const MathTabs &T, TaskSink &s, int read, const AlnReg *a, int n, int extra_flag, i32 *cnt)
{
	plan_xa(o, s, read, a, n, cnt);
	int l = 0, mapq0 = 0;
	for (int k = 0; k < n; ++k) {
		if (a[k].score < o.T || a[k].secondary >= 0) continue;
		int mapq = approx_mapq_d(o, a[k], T);
		if (l && mapq > mapq0) mapq = mapq0;
		if (!l) mapq0 = mapq;
		if (l < 255) add_task(s, read, k, 0, l, k, mapq, extra_flag | (l ? 0x800 : 0)); else s.ovf = true;
		++l;
	}
	s.lines = l;
}
SSQ_HD void plan_single(const ssq_opts_t &o, const MathTabs &T, int read, AlnReg *a, int n, i64 id, TaskSink &s, ReadMeta &m, i32 *cnt)
{
	mark_primary_d(o, n, a, id, cnt);
	plan_reg2sam(o, T, s, read, a, n, 0, cnt);
	m.n_tasks = (u32)s.n; m.n_lines = (u32)s.lines; m.extra_flag = 0; m.mode = 1; m.has_hdr = 0;
}
// mem_sam_pe after the mate rescue.  a[i]/n[i]: region lists of the two ends; s[i], m[i]: their task sinks and records; v: scratch
// for mem_pair_d; cnt[i]: n[i] scratch ints
SSQ_HD void plan_pair(const ssq_opts_t &o, const DevIndex &ix, const MathTabs &T, const PeStat *pes, int p, AlnReg *a[2], const int n[2], i64 id,
                      TaskSink s[2], ReadMeta m[2], P64 *v, i32 *cnt[2])
{
	int z[2] = {0, 0}, osc = 0, subo = 0, n_sub = 0, extra_flag = 1;
	mark_primary_d(o, n[0], a[0], id << 1 | 0, cnt[0]);
	mark_primary_d(o, n[1], a[1], id << 1 | 1, cnt[1]);
	bool pairing = false;
	if (n[0] && n[1] && (osc = mem_pair_d(o, ix, T, pes, a, n, id, &subo, &n_sub, z, v)) > 0) {
		bool multi = false;
		for (int i = 0; i < 2; ++i) for (int j = 1; j < n[i]; ++j) if (a[i][j].secondary < 0 && a[i][j].score >= o.T) { multi = true; break; }
		if (!multi) {
			int q_pe, score_un, q_se[2];
			pairing = true;
			score_un = a[0][0].score + a[1][0].score - o.pen_unpaired;
			subo = subo > score_un ? subo : score_un;
			q_pe = RAW_MAPQ(osc - subo, o.a);
			if (n_sub > 0) q_pe -= tab_lg4343(T, n_sub);
			if (q_pe < 0) q_pe = 0;
			if (q_pe > 60) q_pe = 60;
			q_pe = (int)(q_pe * (1. - .5 * (a[0][0].frac_rep + a[1][0].frac_rep)) + .499);
			if (osc > score_un) {
				AlnReg *c[2] = {&a[0][z[0]], &a[1][z[1]]};
				for (int i = 0; i < 2; ++i) {
					if (c[i]->secondary >= 0) { c[i]->sub = a[i][c[i]->secondary].score; c[i]->secondary = -2; }
					q_se[i] = approx_mapq_d(o, *c[i], T);
				}
				q_se[0] = q_se[0] > q_pe ? q_se[0] : q_pe < q_se[0] + 40 ? q_pe : q_se[0] + 40;
				q_se[1] = q_se[1] > q_pe ? q_se[1] : q_pe < q_se[1] + 40 ? q_pe : q_se[1] + 40;
				extra_flag |= 2;
				q_se[0] = q_se[0] < RAW_MAPQ(c[0]->score - c[0]->csub, o.a) ? q_se[0] : RAW_MAPQ(c[0]->score - c[0]->csub, o.a);
				q_se[1] = q_se[1] < RAW_MAPQ(c[1]->score - c[1]->csub, o.a) ? q_se[1] : RAW_MAPQ(c[1]->score - c[1]->csub, o.a);
			} else { z[0] = z[1] = 0; q_se[0] = approx_mapq_d(o, a[0][0], T); q_se[1] = approx_mapq_d(o, a[1][0], T); }
			for (int i = 0; i < 2; ++i) {
				const int k = a[i][z[i]].secondary_all;
				if (k >= 0 && k < n[i]) {
					for (int j = 0; j < n[i]; ++j) if (a[i][j].secondary_all == k || j == k) a[i][j].secondary_all = z[i];
					a[i][z[i]].secondary_all = -1;
				}
			}
			for (int i = 0; i < 2; ++i) {
				const int read = 2 * p + i;
				plan_xa(o, s[i], read, a[i], n[i], cnt[i]);
				add_task(s[i], read, z[i], 0, 0, z[i], q_se[i], 0x40 << i | extra_flag);
				m[i].n_tasks = (u32)s[i].n; m[i].n_lines = 1; m[i].extra_flag = extra_flag; m[i].mode = 0; m[i].has_hdr = 0;
			}
		}
	}
	if (!pairing) {
		int ef = 1;
		for (int i = 0; i < 2; ++i) { // mate header: the best hit if above T, else unmapped
			m[i].has_hdr = 0;
			if (n[i] && a[i][0].score >= o.T) { m[i].has_hdr = 1; add_task(s[i], 2 * p + i, 0, 2, 0, 0, 0, 0); }
		}
		if (n[0] && n[1] && a[0][0].score >= o.T && a[1][0].score >= o.T && a[0][0].rid == a[1][0].rid) {
			i64 dist;
			const int d = infer_dir(ix.l_pac, a[0][0].rb, a[1][0].rb, &dist);
			if (!pes[d].failed && dist >= pes[d].low && dist <= pes[d].high) ef |= 2;
		}
		for (int i = 0; i < 2; ++i) {
			plan_reg2sam(o, T, s[i], 2 * p + i, a[i], n[i], (0x40 << i) | 1 | ef, cnt[i]);
			m[i].n_tasks = (u32)s[i].n; m[i].n_lines = (u32)s[i].lines; m[i].extra_flag = (0x40 << i) | 1 | ef; m[i].mode = 1;
		}
	}
}

// ================================================================================ text ====
template <bool W> struct Sink { char *p; size_t n; };
template <bool W> SSQ_HD void sput(Sink<W> &s, char c) { if (W) s.p[s.n] = c; ++s.n; }
template <bool W> SSQ_HD void sputs(Sink<W> &s, const char *t, int len) { if (W) for (int i = 0; i < len; ++i) s.p[s.n + i] = t[i]; s.n += len; }
template <bool W> SSQ_HD void sputz(Sink<W> &s, const char *t) { for (; *t; ++t) sput(s, *t); }
template <bool W> SSQ_HD void sputn(Sink<W> &s, long long v) // == "%lld"
{
	char b[24]; int n = 24;
	unsigned long long u = v < 0 ? 0ULL - (unsigned long long)v : (unsigned long long)v;
	do { b[--n] = (char)('0' + u % 10); u /= 10; } while (u);
	if (v < 0) b[--n] = '-';
	sputs(s, b + n, 24 - n);
}

struct LineV { // one alignment as mem_aln2sam sees it
	i64 pos; i32 rid, flag, is_rev, mapq, NM, score, sub; const u32 *cig; i32 n_cig; const char *md; i32 md_len; i32 reg_idx;
};
SSQ_HD void linev_unmapped(LineV &l) { l.pos = -1; l.rid = -1; l.flag = 0; l.is_rev = 0; l.mapq = 0; l.NM = 0; l.score = 0; l.sub = 0; l.cig = 0; l.n_cig = 0; l.md = 0; l.md_len = 0; l.reg_idx = -1; }
SSQ_HD int cig_rlen(const u32 *c, int n) { int l = 0; for (int k = 0; k < n; ++k) { const int op = c[k] & 0xf; if (op == 0 || op == 2) l += c[k] >> 4; } return l; }

struct TextCtx { // everything the text stage needs about the batch
	const char *ctg_names; const u32 *ctg_name_off; // contig names, concatenated
	const char *names; const u32 *name_off;          // read names
	const uint8_t *seq; const u64 *read_off;          // base codes
	const char *qual;                                 // same offsets as seq; null = no qualities
	const char *cmt; const u32 *cmt_off;              // FASTQ comments (-C); null = none
	const char *rg_id; i32 rg_len;
};
template <bool W> SSQ_HD void put_ctg(Sink<W> &s, const TextCtx &c, int rid) { sputs(s, c.ctg_names + c.ctg_name_off[rid], (int)(c.ctg_name_off[rid + 1] - c.ctg_name_off[rid])); }

// the patched view of a line and of its mate (mem_aln2sam patches copies: an unmapped end takes the other end's coordinates)
struct Patched { i64 pos, mpos; i32 rid, mrid, flag, is_rev, m_is_rev; bool cig_shown, mcig_shown; };
SSQ_HD Patched patch_line(const LineV &p0, const LineV *m)
{
	Patched v;
	v.pos = p0.pos; v.rid = p0.rid; v.flag = p0.flag; v.is_rev = p0.is_rev; v.cig_shown = p0.n_cig > 0;
	v.mpos = m ? m->pos : -1; v.mrid = m ? m->rid : -1; v.m_is_rev = m ? m->is_rev : 0; v.mcig_shown = m ? m->n_cig > 0 : false;
	v.flag |= m ? 0x1 : 0;
	v.flag |= v.rid < 0 ? 0x4 : 0;
	v.flag |= m && v.mrid < 0 ? 0x8 : 0;
	if (v.rid < 0 && m && v.mrid >= 0) { v.rid = v.mrid; v.pos = v.mpos; v.is_rev = v.m_is_rev; v.cig_shown = false; }
	if (m && v.mrid < 0 && v.rid >= 0) { v.mrid = v.rid; v.mpos = v.pos; v.m_is_rev = v.is_rev; v.mcig_shown = false; }
	v.flag |= v.is_rev ? 0x10 : 0;
	v.flag |= m && v.m_is_rev ? 0x20 : 0;
	return v;
}
SSQ_HD int printed_flag(const Patched &v) { return (v.flag & 0xffff) | (v.flag & 0x10000 ? 0x100 : 0); }

// extras appended by the fused samblaster stage: flag bits to OR in (0x400), MC/MQ tags, QNAME suffix of the splitter stream
struct SbExtra { i32 or_flag; bool tags; const u32 *mc_cig; i32 mc_n; i32 mq; char suffix; };

// one record.  list[0..n_list): the read's lines (list[which] is written); xa tasks: the read's task slice, outs/cigs addressed
// through the callbacks below are supplied by the caller as arrays indexed by task
struct XaSrc { const PTask *tk; int n_tk; const struct AlnOut *outs; const u32 *cigs; int tk_base; };
// SA:Z — the other non-secondary lines of the read; XA:Z — the alternative hits whose owner is the region a line was built from
template <class LS> SSQ_HD bool has_sa(const LS &list, int n_list, int which) { for (int i = 0; i < n_list; ++i) if (i != which && !(list(i).flag & 0x100)) return true; return false; }
template <bool W, class LS>
SSQ_HD void put_sa(Sink<W> &str, const TextCtx &c, const LS &list, int n_list, int which)
{
	for (int i = 0; i < n_list; ++i) {
		if (i == which) continue;
		const LineV r = list(i);
		if (r.flag & 0x100) continue;
		put_ctg(str, c, r.rid); sput(str, ',');
		sputn(str, r.pos + 1); sput(str, ',');
		sput(str, "+-"[r.is_rev]); sput(str, ',');
		for (int k = 0; k < r.n_cig; ++k) { sputn(str, r.cig[k] >> 4); sput(str, "MIDSH"[r.cig[k] & 0xf]); }
		sput(str, ','); sputn(str, r.mapq);
		sput(str, ','); sputn(str, r.NM);
		sput(str, ';');
	}
}
SSQ_HD bool has_xa(const XaSrc &xa, int reg_idx) { for (int t = 0; t < xa.n_tk; ++t) if (xa.tk[t].kind == 1 && xa.tk[t].xa_owner == reg_idx) return true; return false; }
template <bool W>
SSQ_HD void put_xa(Sink<W> &str, const TextCtx &c, const XaSrc &xa, int reg_idx)
{
	for (int t = 0; t < xa.n_tk; ++t) {
		if (xa.tk[t].kind != 1 || xa.tk[t].xa_owner != reg_idx) continue;
		const AlnOut &ao = xa.outs[xa.tk_base + t];
		const u32 *cg = xa.cigs + (size_t)(xa.tk_base + t) * CIG_CAP;
		put_ctg(str, c, ao.rid); sput(str, ','); sput(str, "+-"[ao.is_rev]); sputn(str, ao.pos + 1); sput(str, ',');
		for (int k = 0; k < ao.n_cigar; ++k) { sputn(str, cg[k] >> 4); sput(str, "MIDSHN"[cg[k] & 0xf]); }
		sput(str, ','); sputn(str, ao.NM); sput(str, ';');
	}
}
// LS: the read's lines, `LineV operator()(int i) const` (lines are fetched on demand: only SA tags look at the other lines)
template <bool W, class LS>
SSQ_HD void sam_line(Sink<W> &str, const TextCtx &c, int read, const LS &list, int n_list, int which, const LineV *m, const XaSrc &xa, const SbExtra *sb)
{
	const LineV p = list(which);
	const Patched v = patch_line(p, m);
	const int l_seq = (int)(c.read_off[read + 1] - c.read_off[read]);
	const uint8_t *sq = c.seq + c.read_off[read];
	sputs(str, c.names + c.name_off[read], (int)(c.name_off[read + 1] - c.name_off[read]));
	if (sb && sb->suffix) { sput(str, '_'); sput(str, sb->suffix); }
	sput(str, '\t');
	sputn(str, printed_flag(v) | (sb ? sb->or_flag : 0)); sput(str, '\t');
	if (v.rid >= 0) {
		put_ctg(str, c, v.rid); sput(str, '\t');
		sputn(str, v.pos + 1); sput(str, '\t');
		sputn(str, p.mapq); sput(str, '\t');
		if (v.cig_shown) {
			for (int i = 0; i < p.n_cig; ++i) {
				int op = p.cig[i] & 0xf;
				if (op == 3 || op == 4) op = which ? 4 : 3;
				sputn(str, p.cig[i] >> 4); sput(str, "MIDSH"[op]);
			}
		} else sput(str, '*');
	} else sputs(str, "*\t0\t0\t*", 7);
	sput(str, '\t');
	if (m && v.mrid >= 0) {
		if (v.rid == v.mrid) sput(str, '='); else put_ctg(str, c, v.mrid);
		sput(str, '\t');
		sputn(str, v.mpos + 1); sput(str, '\t');
		if (v.rid == v.mrid) {
			const i64 p0 = v.pos + (v.is_rev ? (v.cig_shown ? cig_rlen(p.cig, p.n_cig) : 0) - 1 : 0), p1 = v.mpos + (v.m_is_rev ? (v.mcig_shown ? cig_rlen(m->cig, m->n_cig) : 0) - 1 : 0);
			if (!v.mcig_shown || !v.cig_shown) sput(str, '0');
			else sputn(str, -(p0 - p1 + (p0 > p1 ? 1 : p0 < p1 ? -1 : 0)));
		} else sput(str, '0');
	} else sputs(str, "*\t0\t0", 5);
	sput(str, '\t');
	if (v.flag & 0x100) sputs(str, "*\t*", 3);
	else {
		int qb = 0, qe = l_seq;
		if (v.cig_shown && which) {
			const int c0 = p.cig[0] & 0xf, c1 = p.cig[p.n_cig - 1] & 0xf;
			if (!v.is_rev) { if (c0 == 4 || c0 == 3) qb += p.cig[0] >> 4; if (c1 == 4 || c1 == 3) qe -= p.cig[p.n_cig - 1] >> 4; }
			else { if (c0 == 4 || c0 == 3) qe -= p.cig[0] >> 4; if (c1 == 4 || c1 == 3) qb += p.cig[p.n_cig - 1] >> 4; }
		}
		const char *ql = c.qual ? c.qual + c.read_off[read] : 0;
		if (!v.is_rev) {
			if (W) for (int i = qb; i < qe; ++i) str.p[str.n + (i - qb)] = "ACGTN"[sq[i]];
			str.n += qe - qb;
			sput(str, '\t');
			if (ql) sputs(str, ql + qb, qe - qb); else sput(str, '*');
		} else {
			if (W) for (int i = qe - 1; i >= qb; --i) str.p[str.n + (qe - 1 - i)] = "TGCAN"[sq[i]];
			str.n += qe - qb;
			sput(str, '\t');
			if (ql) { if (W) for (int i = qe - 1; i >= qb; --i) str.p[str.n + (qe - 1 - i)] = ql[i]; str.n += qe - qb; } else sput(str, '*');
		}
	}
	if (v.cig_shown) { sputs(str, "\tNM:i:", 6); sputn(str, p.NM); sputs(str, "\tMD:Z:", 6); sputs(str, p.md, p.md_len); }
	if (p.score >= 0) { sputs(str, "\tAS:i:", 6); sputn(str, p.score); }
	if (p.sub >= 0) { sputs(str, "\tXS:i:", 6); sputn(str, p.sub); }
	if (c.rg_len) { sputs(str, "\tRG:Z:", 6); sputs(str, c.rg_id, c.rg_len); }
	if (!(v.flag & 0x100) && has_sa(list, n_list, which)) { sputs(str, "\tSA:Z:", 6); put_sa(str, c, list, n_list, which); }
	if (has_xa(xa, p.reg_idx)) { sputs(str, "\tXA:Z:", 6); put_xa(str, c, xa, p.reg_idx); }
	if (c.cmt && c.cmt_off[read + 1] > c.cmt_off[read]) { sput(str, '\t'); sputs(str, c.cmt + c.cmt_off[read], (int)(c.cmt_off[read + 1] - c.cmt_off[read])); }
	if (sb && sb->tags) {
		sputs(str, "\tMC:Z:", 6);
		if (sb->mc_n > 0) for (int k = 0; k < sb->mc_n; ++k) { int op = sb->mc_cig[k] & 0xf; if (op == 4) op = 3; sputn(str, sb->mc_cig[k] >> 4); sput(str, "MIDSH"[op]); } else sput(str, '*');
		sputs(str, "\tMQ:i:", 6); sputn(str, sb->mq);
	}
	sput(str, '\n');
}


// =================================================================================== BAM ====
// The records of the three streams as BAM (SURVEY.md §8 f1): what `sambamba view -S -f bam` makes of the SAM text, encoded
// straight from the structured records.  Layout: speedseq/src/samtools-1.3.1/htslib-1.3.1/sam.c:443-467 (bam_write1 /
// the in-memory record), bin: htslib/hts.h:580-586 (hts_reg2bin), integer tags take the smallest type that holds the value.
// Parity is pinned on the reference's OWN tool: tests/golden/ex_bam_*.gz were produced by speedseq/src/sambamba (v0.5.9)
// from the oracle's SAM of the example reads (tests/golden/make_bam_golden.py).
template <bool W> SSQ_HD void bput32(Sink<W> &s, u32 v) { if (W) { s.p[s.n] = (char)v; s.p[s.n + 1] = (char)(v >> 8); s.p[s.n + 2] = (char)(v >> 16); s.p[s.n + 3] = (char)(v >> 24); } s.n += 4; }
template <bool W> SSQ_HD void bput16(Sink<W> &s, u32 v) { if (W) { s.p[s.n] = (char)v; s.p[s.n + 1] = (char)(v >> 8); } s.n += 2; }
template <bool W> SSQ_HD void bput_int_tag(Sink<W> &s, char t0, char t1, long long v)
{
	sput(s, t0); sput(s, t1);
	if (v < 0) { if (v >= -128) { sput(s, 'c'); sput(s, (char)v); } else if (v >= -32768) { sput(s, 's'); bput16(s, (u32)v); } else { sput(s, 'i'); bput32(s, (u32)v); } }
	else if (v <= 255) { sput(s, 'C'); sput(s, (char)v); } else if (v <= 65535) { sput(s, 'S'); bput16(s, (u32)v); } else { sput(s, 'I'); bput32(s, (u32)v); }
}
SSQ_HD int bam_reg2bin(i64 beg, i64 end)
{
	--end;
	if (beg >> 14 == end >> 14) return (int)(((1 << 15) - 1) / 7 + (beg >> 14));
	if (beg >> 17 == end >> 17) return (int)(((1 << 12) - 1) / 7 + (beg >> 17));
	if (beg >> 20 == end >> 20) return (int)(((1 << 9) - 1) / 7 + (beg >> 20));
	if (beg >> 23 == end >> 23) return (int)(((1 << 6) - 1) / 7 + (beg >> 23));
	if (beg >> 26 == end >> 26) return (int)(((1 << 3) - 1) / 7 + (beg >> 26));
	return 0;
}
// coordinate-sort key of a line: (tid, pos, reverse strand), records without a reference last; equal keys keep input order
SSQ_HD u64 bam_sort_key(const Patched &v) { return v.rid < 0 ? ~0ull : ((u64)(u32)v.rid << 34 | (u64)(v.pos + 1) << 1 | (u64)(v.is_rev ? 1 : 0)); }

// one record (block_size included).  blank: SEQ and QUAL are '*' (what speedseq's gawk step makes of the side streams, speedseq:443,446).
// *bad is set when a -C comment is not TAG:TYPE:VALUE with TYPE in {Z, i, A}
template <bool W, class LS>
SSQ_HD void bam_record(Sink<W> &str, const TextCtx &c, int read, const LS &list, int n_list, int which, const LineV *m, const XaSrc &xa, const SbExtra *sb, bool blank, int *bad)
{
	const LineV p = list(which);
	const Patched v = patch_line(p, m);
	const int l_read = (int)(c.read_off[read + 1] - c.read_off[read]);
	const uint8_t *sq = c.seq + c.read_off[read];
	const int flag = printed_flag(v) | (sb ? sb->or_flag : 0);
	const size_t at0 = str.n;
	bput32(str, 0); // block_size, patched below
	const int n_cig = v.cig_shown ? p.n_cig : 0;
	const i64 pos = v.rid >= 0 ? v.pos : -1;
	const int rlen = n_cig ? cig_rlen(p.cig, p.n_cig) : 0;
	const i64 end = (flag & 4) || rlen == 0 ? pos + 1 : pos + rlen;
	const int name_l = (int)(c.name_off[read + 1] - c.name_off[read]) + (sb && sb->suffix ? 2 : 0);
	int qb = 0, qe = l_read;
	if (v.cig_shown && which) {
		const int c0 = p.cig[0] & 0xf, c1 = p.cig[p.n_cig - 1] & 0xf;
		if (!v.is_rev) { if (c0 == 4 || c0 == 3) qb += p.cig[0] >> 4; if (c1 == 4 || c1 == 3) qe -= p.cig[p.n_cig - 1] >> 4; }
		else { if (c0 == 4 || c0 == 3) qe -= p.cig[0] >> 4; if (c1 == 4 || c1 == 3) qb += p.cig[p.n_cig - 1] >> 4; }
	}
	const int l_seq = (blank || (v.flag & 0x100)) ? 0 : qe - qb;
	bput32(str, (u32)v.rid); bput32(str, (u32)pos);
	sput(str, (char)(name_l + 1)); sput(str, (char)(v.rid >= 0 ? p.mapq : 0)); bput16(str, (u32)bam_reg2bin(pos, end));
	bput16(str, (u32)n_cig); bput16(str, (u32)flag); bput32(str, (u32)l_seq);
	const bool has_mate = m && v.mrid >= 0;
	bput32(str, (u32)(has_mate ? v.mrid : -1)); bput32(str, (u32)(has_mate ? v.mpos : -1));
	i64 tlen = 0;
	if (has_mate && v.rid == v.mrid && v.mcig_shown && v.cig_shown) {
		const i64 p0 = v.pos + (v.is_rev ? cig_rlen(p.cig, p.n_cig) - 1 : 0), p1 = v.mpos + (v.m_is_rev ? cig_rlen(m->cig, m->n_cig) - 1 : 0);
		tlen = -(p0 - p1 + (p0 > p1 ? 1 : p0 < p1 ? -1 : 0));
	}
	bput32(str, (u32)tlen);
	sputs(str, c.names + c.name_off[read], (int)(c.name_off[read + 1] - c.name_off[read]));
	if (sb && sb->suffix) { sput(str, '_'); sput(str, sb->suffix); }
	sput(str, 0);
	for (int i = 0; i < n_cig; ++i) {
		int op = p.cig[i] & 0xf;
		if (op == 3 || op == 4) op = which ? 4 : 3;
		bput32(str, (p.cig[i] >> 4) << 4 | (u32)(op == 3 ? 4 : op == 4 ? 5 : op)); // internal 3 = S, 4 = H -> BAM 4, 5
	}
	if (l_seq) {
		const char *ql = c.qual ? c.qual + c.read_off[read] : 0;
		for (int k = 0; k < l_seq; k += 2) { // 4 bits per base: A 1, C 2, G 4, T 8, N 15
			int nib[2] = {0, 0};
			for (int h = 0; h < 2 && k + h < l_seq; ++h) { const int b = !v.is_rev ? sq[qb + k + h] : (sq[qe - 1 - k - h] < 4 ? 3 - sq[qe - 1 - k - h] : 4); nib[h] = b == 0 ? 1 : b == 1 ? 2 : b == 2 ? 4 : b == 3 ? 8 : 15; }
			sput(str, (char)(nib[0] << 4 | nib[1]));
		}
		for (int k = 0; k < l_seq; ++k) sput(str, ql ? (char)((!v.is_rev ? ql[qb + k] : ql[qe - 1 - k]) - 33) : (char)0xff);
	}
	if (v.cig_shown) { bput_int_tag(str, 'N', 'M', p.NM); sputs(str, "MDZ", 3); sputs(str, p.md, p.md_len); sput(str, 0); }
	if (p.score >= 0) bput_int_tag(str, 'A', 'S', p.score);
	if (p.sub >= 0) bput_int_tag(str, 'X', 'S', p.sub);
	if (c.rg_len) { sputs(str, "RGZ", 3); sputs(str, c.rg_id, c.rg_len); sput(str, 0); }
	if (!(v.flag & 0x100) && has_sa(list, n_list, which)) { sputs(str, "SAZ", 3); put_sa(str, c, list, n_list, which); sput(str, 0); }
	if (has_xa(xa, p.reg_idx)) { sputs(str, "XAZ", 3); put_xa(str, c, xa, p.reg_idx); sput(str, 0); }
	if (c.cmt && c.cmt_off[read + 1] > c.cmt_off[read]) { // -C: the FASTQ comment holds tab-separated TAG:TYPE:VALUE fields
		const char *t = c.cmt + c.cmt_off[read]; const int n = (int)(c.cmt_off[read + 1] - c.cmt_off[read]);
		int i = 0;
		while (i < n) {
			int e = i; while (e < n && t[e] != '\t') ++e;
			if (e - i >= 5 && t[i + 2] == ':' && t[i + 4] == ':' && (t[i + 3] == 'Z' || t[i + 3] == 'A' || t[i + 3] == 'i')) {
				if (t[i + 3] == 'Z') { sput(str, t[i]); sput(str, t[i + 1]); sput(str, 'Z'); sputs(str, t + i + 5, e - i - 5); sput(str, 0); }
				else if (t[i + 3] == 'A') { sput(str, t[i]); sput(str, t[i + 1]); sput(str, 'A'); sput(str, e - i > 5 ? t[i + 5] : ' '); }
				else { long long x = 0; bool neg = false; int k = i + 5; if (k < e && (t[k] == '-' || t[k] == '+')) { neg = t[k] == '-'; ++k; } for (; k < e; ++k) x = x * 10 + (t[k] - '0'); bput_int_tag(str, t[i], t[i + 1], neg ? -x : x); }
			} else if (bad) *bad = 1;
			i = e + 1;
		}
	}
	if (sb && sb->tags) {
		sputs(str, "MCZ", 3);
		if (sb->mc_n > 0) for (int k = 0; k < sb->mc_n; ++k) { int op = sb->mc_cig[k] & 0xf; if (op == 4) op = 3; sputn(str, sb->mc_cig[k] >> 4); sput(str, "MIDSH"[op]); } else sput(str, '*');
		sput(str, 0);
		bput_int_tag(str, 'M', 'Q', sb->mq);
	}
	if (W) { const u32 bs = (u32)(str.n - at0 - 4); str.p[at0] = (char)bs; str.p[at0 + 1] = (char)(bs >> 8); str.p[at0 + 2] = (char)(bs >> 16); str.p[at0 + 3] = (char)(bs >> 24); }
}

// ============================================================================ samblaster ====
#define SB_PAD 500
struct SbOpts { i32 enabled, excludeDups, addMateTags, maxSplitCount, minNonOverlap, minIndelSize, maxUnmappedBases, removeDups, want_split, want_disc; };
struct SbGeom { i32 raLen, qaLen, sclip, eclip, SQO, EQO; i64 rapos, pos; }; // calcOffsets of a printed line
// printed CIGAR of a line: ops 3/4 are both clips; `shown` false = '*'
SSQ_HD SbGeom sb_geometry(const u32 *cig, int n_cig, bool shown, i64 printed_pos1 /* POS field */, bool rev)
{
	SbGeom g; g.raLen = g.qaLen = g.sclip = g.eclip = 0;
	bool first = true;
	if (shown) for (int k = 0; k < n_cig; ++k) {
		const int op = cig[k] & 0xf, len = (int)(cig[k] >> 4);
		if (op == 0) { g.raLen += len; g.qaLen += len; first = false; }
		else if (op == 3 || op == 4) { if (first) g.sclip += len; else g.eclip += len; }
		else if (op == 2) g.raLen += len;
		else if (op == 1) g.qaLen += len;
	}
	g.rapos = printed_pos1;
	if (!rev) { g.pos = g.rapos - g.sclip; g.SQO = g.sclip; g.EQO = g.sclip + g.qaLen - 1; }
	else { g.pos = g.rapos + g.raLen + g.eclip - 1; g.SQO = g.eclip; g.EQO = g.eclip + g.qaLen - 1; }
	g.pos += SB_PAD;
	return g;
}
// a block's primary line as samblaster reads it back from the text
struct SbLine { i32 flag, rid; bool shown; const u32 *cig; i32 n_cig; i64 pos1; };
// signature of a pair block (both primaries present).  sb_off[rid] = offset of contig rid in samblaster's padded coordinate
// space (sum of LN + 2*PAD + 1 over the earlier @SQ lines).  Returns valid; *disc = the pair is discordant
SSQ_HD bool sb_pair_signature(const SbLine &f, const SbLine &s, const i64 *sb_off, u64 *k1, u64 *k2, bool *disc)
{
	*disc = false; *k1 = *k2 = 0;
	if ((f.flag & 0x4) && (s.flag & 0x4)) return false;
	const bool orphan = (f.flag & 0x4) || (s.flag & 0x4);
	const SbLine *first = &f, *second = &s;
	if (!(f.flag & 0x4) && (s.flag & 0x4)) { first = &s; second = &f; } // the unmapped end goes first
	const SbGeom g2 = sb_geometry(second->cig, second->n_cig, second->shown, second->pos1, (second->flag & 0x10) != 0);
	i64 pos_a = 0, pos_b = g2.pos; int seq_a = -1, seq_b = second->rid;
	if (!orphan) {
		const SbGeom g1 = sb_geometry(first->cig, first->n_cig, first->shown, first->pos1, (first->flag & 0x10) != 0);
		pos_a = g1.pos; seq_a = first->rid;
		bool swap;
		if (pos_a > pos_b) swap = true; else if (pos_a < pos_b) swap = false;
		else if (seq_a > seq_b) swap = true; else if (seq_a < seq_b) swap = false;
		else if ((first->flag & 0x10) == (second->flag & 0x10)) swap = false;
		else swap = (first->flag & 0x10) && !(second->flag & 0x10);
		if (swap) { const SbLine *t = first; first = second; second = t; const i64 tp = pos_a; pos_a = pos_b; pos_b = tp; const int ts = seq_a; seq_a = seq_b; seq_b = ts; }
	}
	const u64 a = orphan ? 0 : (u64)(sb_off[seq_a] + pos_a) + 1, b = (u64)(sb_off[seq_b] + pos_b) + 1;
	*k1 = a << 1 | ((first->flag & 0x10) ? 1 : 0);
	*k2 = b << 1 | ((second->flag & 0x10) ? 1 : 0);
	*disc = !orphan && !(first->flag & 0x2);
	return true;
}
// signature of a block with a single primary line (single-end read, or one end missing)
SSQ_HD bool sb_lone_signature(const SbLine &only, const i64 *sb_off, u64 *k1, u64 *k2)
{
	*k1 = *k2 = 0;
	if ((only.flag & 0x1) && ((only.flag & 0x4) || !(only.flag & 0x8))) return false;
	if (only.flag & 0x4) return false;
	const SbGeom g = sb_geometry(only.cig, only.n_cig, only.shown, only.pos1, (only.flag & 0x10) != 0);
	*k1 = 0; // the absent mate: position 0, forward
	*k2 = ((u64)(sb_off[only.rid] + g.pos) + 1) << 1 | ((only.flag & 0x10) ? 1 : 0);
	return true;
}
// splitter test over the lines of one read side (primary + supplementary, mapped): geometry per line, result bit per line.
// n <= 64; returns a bitmask of the lines that are splitters
struct SbSplitLine { SbGeom g; i32 flag, rid; };
SSQ_HD u64 sb_splitters(const SbOpts &o, SbSplitLine *l, int count)
{
	if (count < 2 || count > o.maxSplitCount || count > 64) return 0;
	int ord[64];
	for (int i = 0; i < count; ++i) ord[i] = i;
	for (int i = 1; i < count; ++i) for (int j = i; j > 0 && l[ord[j]].g.SQO < l[ord[j - 1]].g.SQO; --j) { const int t = ord[j]; ord[j] = ord[j - 1]; ord[j - 1] = t; } // stable; SQO ties cannot occur among non-secondary lines
	u64 mask = 0;
	for (int i = 1; i < count; ++i) {
		const SbSplitLine &left = l[ord[i - 1]], &right = l[ord[i]];
		int overlap = 1 + (left.g.EQO < right.g.EQO ? left.g.EQO : right.g.EQO) - (left.g.SQO > right.g.SQO ? left.g.SQO : right.g.SQO);
		if (overlap < 0) overlap = 0;
		const int alen1 = 1 + left.g.EQO - left.g.SQO, alen2 = 1 + right.g.EQO - right.g.SQO;
		const int mno = alen1 - overlap < alen2 - overlap ? alen1 - overlap : alen2 - overlap;
		if (mno < o.minNonOverlap) continue;
		if (left.rid == right.rid && (left.flag & 0x10) == (right.flag & 0x10)) {
			const int sd_l = (int)(left.g.rapos - left.g.sclip), ed_l = (int)((left.g.rapos + left.g.raLen) - (left.g.sclip + left.g.qaLen));
			const int sd_r = (int)(right.g.rapos - right.g.sclip), ed_r = (int)((right.g.rapos + right.g.raLen) - (right.g.sclip + right.g.qaLen));
			const int ins = (left.flag & 0x10) ? ed_r - sd_l : ed_l - sd_r;
			const int desert = right.g.SQO - left.g.EQO - 1;
			if ((ins < 0 ? -ins : ins) < o.minIndelSize || (desert > 0 && desert - (ins > 0 ? ins : 0) > o.maxUnmappedBases)) continue;
		}
		mask |= 1ull << ord[i - 1] | 1ull << ord[i];
	}
	return mask;
}

// =============================================================== per-thread bodies of the pipeline ====
// The kernels of ssq_pipe.cu are loops over these bodies (one read / pair / task per thread); tests/hostsim runs the same
// bodies in plain for-loops.  All pointers are device pointers in the product.
struct PipeView {
	DevIndex ix; ssq_opts_t opt; MathTabs T; SbOpts sb; TextCtx tc;
	i32 n_reads, paired; i64 n_processed;
	// stage-0 regions of read r (ssq_batch_run): regs[task_off[r] .. +n_regs[r])
	const u64 *task_off; const u32 *n_regs; const RegCand *regs;
	// region lists with room for rescued hits: areg[areg_off[r] .. +n_areg[r]), capacity areg_off[r+1] - areg_off[r]
	const u64 *areg_off; AlnReg *areg; u32 *n_areg;
	const PeStat *pes; u32 *hist; i32 hist_n; // insert-size histogram: hist[dir * hist_n + isize]
	// planning: task slots of read r at tslots[tslot_off[r] ..) (capacity 2 * n_areg[r] + 1), per-read record, scratch
	const u64 *tslot_off; PTask *tslots; ReadMeta *meta; P64 *pv; i32 *xcnt;
	// compact tasks: read r owns tasks[tk_base[r] .. tk_base[r] + meta[r].n_tasks); results per task
	const u64 *tk_base; PTask *tasks; AlnOut *outs; u32 *cigs; char *mds;
	// samblaster (block = pair, or single read when !paired)
	const i64 *sb_off; u64 *k1, *k2; uint8_t *valid, *dup, *disc; u64 *split_mask;
	// text: per-read byte counts / offsets of the three streams (0 main, 1 splitters, 2 discordants) and the buffers
	u64 *len[3]; const u64 *off[3]; char *text[3];
	// BAM (optional): lines are numbered read by read (line_base), sorted by coordinate (perm: sorted position -> line); per stream the
	// byte size of every line (0 = not in the stream) and, after the sort, the offset of every sorted position
	const u64 *line_base; u32 *line_read; u64 *bam_key; u64 *bam_size[3]; const u32 *bam_perm; const u64 *bam_off[3]; char *bam[3]; i32 bam_blank_side;
	unsigned long long *cnt; // device-measured work: [0] duplicate blocks, [2] local-SW passes of the mate rescue, [3] their cells (rows x query length), [4] banded-DP cells of CIGAR generation
	i32 *err; // sticky error flags: 1 region-list overflow, 2 task-slot overflow, 4 CIGAR/MD/traceback capacity, 8 rescue window capacity
};
#ifdef __CUDA_ARCH__
#define PIPE_ERR(V, bit) atomicOr((V).err, (bit))
#else
#define PIPE_ERR(V, bit) (*(V).err |= (bit))
#endif

// stage 1: RegCand list -> sorted / de-duplicated / patched AlnReg list
SSQ_HD void body_dedup(const PipeView &V, int r, const AlnScratch &A)
{
	const int n0 = (int)V.n_regs[r];
	AlnReg *a = V.areg + V.areg_off[r];
	for (int i = 0; i < n0; ++i) reg_from_cand(V.regs[V.task_off[r] + i], a[i]);
	V.n_areg[r] = (u32)sort_dedup_patch(V.ix, V.opt, V.tc.seq + V.tc.read_off[r], n0, a, A, V.xcnt + V.areg_off[r]);
}
// stage 2: a pair's vote in the insert-size histogram; returns true when it voted
SSQ_HD bool body_pestat(const PipeView &V, int p, int *dir, i64 *is)
{
	return pestat_pair(V.opt, V.ix.l_pac, V.areg + V.areg_off[2 * p], (int)V.n_areg[2 * p], V.areg + V.areg_off[2 * p + 1], (int)V.n_areg[2 * p + 1], dir, is);
}
// does end i of pair p trigger at least one rescue alignment?  (mem_matesw's skip test against the mate's CURRENT list; when no
// anchor of either end triggers one, the lists never change and the whole pair needs no work)
SSQ_HD bool rescue_wanted(const PipeView &V, int p)
{
	const i64 l_pac = V.ix.l_pac;
	for (int i = 0; i < 2; ++i) {
		const AlnReg *a = V.areg + V.areg_off[2 * p + i], *ma = V.areg + V.areg_off[2 * p + !i];
		const int na = (int)V.n_areg[2 * p + i], nm = (int)V.n_areg[2 * p + !i];
		int nb = 0;
		for (int j = 0; j < na && nb < V.opt.max_matesw; ++j) {
			if (!(a[j].score >= a[0].score - V.opt.pen_unpaired)) continue;
			++nb;
			int skip[4];
			for (int r = 0; r < 4; ++r) skip[r] = V.pes[r].failed ? 1 : 0;
			for (int k = 0; k < nm; ++k) {
				i64 dist;
				const int r = infer_dir(l_pac, a[j].rb, ma[k].rb, &dist);
				if (dist >= V.pes[r].low && dist <= V.pes[r].high) skip[r] = 1;
			}
			if (skip[0] + skip[1] + skip[2] + skip[3] != 4) return true;
		}
	}
	return false;
}
// the rescue alignments of pair p the lists, as they are before any rescue, do not skip: their count, and with `out` the tasks
// themselves in replay order (end, snapshot index, orientation).  win_cap: windows beyond it are left to the replay, which reports them
SSQ_HD int rescue_enum(const PipeView &V, int p, RTask *out, u32 slot, int win_cap)
{
	const i64 l_pac = V.ix.l_pac;
	int n = 0;
	for (int i = 0; i < 2; ++i) {
		const AlnReg *a = V.areg + V.areg_off[2 * p + i], *ma = V.areg + V.areg_off[2 * p + !i];
		const int na = (int)V.n_areg[2 * p + i], nm = (int)V.n_areg[2 * p + !i];
		const int l_ms = (int)(V.tc.read_off[2 * p + !i + 1] - V.tc.read_off[2 * p + !i]);
		int nb = 0;
		for (int j = 0; j < na && nb < V.opt.max_matesw && nb < 64; ++j) {
			if (!(a[j].score >= a[0].score - V.opt.pen_unpaired)) continue;
			const int jj = nb++; // index in the snapshot of near-best hits (body_rescue)
			int skip[4];
			for (int r = 0; r < 4; ++r) skip[r] = V.pes[r].failed ? 1 : 0;
			for (int k = 0; k < nm; ++k) {
				i64 dist;
				const int r = infer_dir(l_pac, a[j].rb, ma[k].rb, &dist);
				if (dist >= V.pes[r].low && dist <= V.pes[r].high) skip[r] = 1;
			}
			for (int r = 0; r < 4; ++r) {
				i64 rb, re;
				if (skip[r] || !rescue_window(V.ix, V.opt, V.pes, a[j], l_ms, r, &rb, &re) || re - rb > win_cap) continue;
				if (out) { RTask t; t.slot = slot; t.key = (u32)(i << 16 | jj << 2 | r); t.rb = rb; t.tlen = (i32)(re - rb); t.l_ms = l_ms; out[n] = t; }
				++n;
			}
		}
	}
	return n;
}
// stage 3: mate rescue of one pair (mem_sam_pe's first block).  bbuf: room for 2 x 64 regions (the near-best hits of both ends are
// copied before any list changes, as the reference does)
SSQ_HD void body_rescue(const PipeView &V, int p, AlnReg *bbuf, const MateScratch &M, RCache *rc = 0)
{
	AlnReg *b[2] = {bbuf, bbuf + 64};
	int nb[2] = {0, 0}, na[2];
	AlnReg *a[2];
	for (int i = 0; i < 2; ++i) {
		a[i] = V.areg + V.areg_off[2 * p + i]; na[i] = (int)V.n_areg[2 * p + i];
		for (int j = 0; j < na[i]; ++j)
			if (a[i][j].score >= a[i][0].score - V.opt.pen_unpaired && nb[i] < 64) b[i][nb[i]++] = a[i][j]; // only the first max_matesw (50) are used
	}
	for (int i = 0; i < 2; ++i) {
		const int cap = (int)(V.areg_off[2 * p + !i + 1] - V.areg_off[2 * p + !i]);
		for (int j = 0; j < nb[i] && j < V.opt.max_matesw; ++j) {
			const int before = na[!i];
			if (mate_rescue(V.ix, V.opt, V.pes, b[i][j], (int)(V.tc.read_off[2 * p + !i + 1] - V.tc.read_off[2 * p + !i]), V.tc.seq + V.tc.read_off[2 * p + !i], a[!i], &na[!i], cap, M, V.xcnt + V.areg_off[2 * p + !i], rc, (u32)(i << 16 | j << 2)) < 0) PIPE_ERR(V, 8);
			if (na[!i] >= cap && before < cap) PIPE_ERR(V, 1);
		}
	}
	V.n_areg[2 * p] = (u32)na[0]; V.n_areg[2 * p + 1] = (u32)na[1];
}
// stage 4: primary marking, pairing, MAPQ and the list of alignments to write (unit u = pair when paired, read otherwise)
SSQ_HD void body_plan(const PipeView &V, int u)
{
	if (!V.paired) {
		const int r = u;
		TaskSink s; s.t = V.tslots + V.tslot_off[r]; s.n = 0; s.cap = (int)(V.tslot_off[r + 1] - V.tslot_off[r]); s.lines = 0; s.ovf = false;
		ReadMeta m; m.pad[0] = m.pad[1] = 0;
		plan_single(V.opt, V.T, r, V.areg + V.areg_off[r], (int)V.n_areg[r], V.n_processed + r, s, m, V.xcnt + V.areg_off[r]);
		V.meta[r] = m;
		if (s.ovf) PIPE_ERR(V, 2);
		return;
	}
	const int p = u;
	AlnReg *a[2] = {V.areg + V.areg_off[2 * p], V.areg + V.areg_off[2 * p + 1]};
	const int n[2] = {(int)V.n_areg[2 * p], (int)V.n_areg[2 * p + 1]};
	TaskSink s[2]; ReadMeta m[2]; i32 *cnt[2];
	for (int i = 0; i < 2; ++i) {
		s[i].t = V.tslots + V.tslot_off[2 * p + i]; s[i].n = 0; s[i].cap = (int)(V.tslot_off[2 * p + i + 1] - V.tslot_off[2 * p + i]); s[i].lines = 0; s[i].ovf = false;
		m[i].pad[0] = m[i].pad[1] = 0; m[i].has_hdr = 0;
		cnt[i] = V.xcnt + V.areg_off[2 * p + i];
	}
	plan_pair(V.opt, V.ix, V.T, V.pes, p, a, n, (V.n_processed >> 1) + p, s, m, V.pv + V.areg_off[2 * p], cnt);
	V.meta[2 * p] = m[0]; V.meta[2 * p + 1] = m[1];
	if (s[0].ovf || s[1].ovf) PIPE_ERR(V, 2);
}
// stage 5: position / CIGAR / NM / MD of compact task t
SSQ_HD void body_cigar(const PipeView &V, u64 t, const AlnScratch &A)
{
	const PTask k = V.tasks[t];
	const AlnReg &reg = V.areg[V.areg_off[k.read] + k.reg_idx];
	AlnOut a;
	reg2aln(V.ix, V.opt, (int)(V.tc.read_off[k.read + 1] - V.tc.read_off[k.read]), V.tc.seq + V.tc.read_off[k.read], reg, A, a, V.cigs + t * CIG_CAP, CIG_CAP, V.mds + t * MD_CAP, MD_CAP);
	if (a.n_cigar < 0 || a.n_cigar > CIG_CAP - 2 || a.md_len >= MD_CAP) PIPE_ERR(V, 4);
	V.outs[t] = a;
}

// ---- line access for the text and samblaster stages ----
SSQ_HD LineV line_of_task(const PipeView &V, u64 t)
{
	const PTask &k = V.tasks[t]; const AlnOut &ao = V.outs[t];
	LineV l;
	l.pos = ao.pos; l.rid = ao.rid; l.flag = k.flag | ao.flag; l.is_rev = ao.is_rev; l.mapq = k.mapq; l.NM = ao.NM; l.score = ao.score; l.sub = ao.sub;
	l.cig = V.cigs + t * CIG_CAP; l.n_cig = ao.n_cigar; l.md = V.mds + t * MD_CAP; l.md_len = ao.md_len; l.reg_idx = k.reg_idx;
	return l;
}
SSQ_HD int read_n_lines(const PipeView &V, int r) { return V.meta[r].n_lines ? V.meta[r].n_lines : 1; } // an unaligned read still writes one record
SSQ_HD LineV read_line(const PipeView &V, int r, int i) // the read's lines are the last n_lines tasks of its slice
{
	const ReadMeta &m = V.meta[r];
	if (m.n_lines == 0) { LineV l; linev_unmapped(l); l.flag = 0x4 | m.extra_flag; return l; }
	return line_of_task(V, V.tk_base[r] + m.n_tasks - m.n_lines + i);
}
// what the lines of read r show as their mate (mem_sam_pe: the mate's first line when the pair was written as a pair, else the
// mate's best hit if above T, else an unmapped placeholder)
SSQ_HD LineV mate_header(const PipeView &V, int r)
{
	const int m = r ^ 1;
	const ReadMeta &mm = V.meta[m];
	if (mm.mode == 0) return read_line(V, m, 0);
	if (mm.has_hdr) { LineV l = line_of_task(V, V.tk_base[m]); l.mapq = 0; return l; } // kind-2 task is the first of the slice
	LineV l; linev_unmapped(l); return l;
}
// the primary line of read r as samblaster parses it back from the text
SSQ_HD SbLine sb_primary(const PipeView &V, int r, int *mapq_printed)
{
	const LineV l = read_line(V, r, 0);
	LineV mh; const LineV *m = 0;
	if (V.paired) { mh = mate_header(V, r); m = &mh; }
	const Patched v = patch_line(l, m);
	SbLine s;
	s.flag = printed_flag(v); s.rid = v.rid; s.shown = v.cig_shown; s.cig = l.cig; s.n_cig = l.n_cig; s.pos1 = v.rid >= 0 ? v.pos + 1 : 0;
	*mapq_printed = v.rid >= 0 ? l.mapq : 0;
	return s;
}
// stage 6: samblaster over block u (pair / single read): signature, discordant bit, splitter masks
SSQ_HD void body_sb(const PipeView &V, int u)
{
	int mq;
	u64 k1 = 0, k2 = 0; bool disc = false, valid;
	const int r0 = V.paired ? 2 * u : u, nr = V.paired ? 2 : 1;
	if (V.paired) {
		const SbLine f = sb_primary(V, r0, &mq), s = sb_primary(V, r0 + 1, &mq);
		valid = sb_pair_signature(f, s, V.sb_off, &k1, &k2, &disc);
	} else {
		const SbLine only = sb_primary(V, r0, &mq);
		valid = sb_lone_signature(only, V.sb_off, &k1, &k2);
	}
	V.k1[u] = k1; V.k2[u] = k2; V.valid[u] = valid ? 1 : 0; V.disc[u] = disc ? 1 : 0;
	for (int i = 0; i < nr; ++i) {
		const int r = r0 + i;
		u64 mask = 0;
		const int nl = V.meta[r].n_lines;
		if (V.sb.want_split && V.paired && nl >= 2 && nl <= V.sb.maxSplitCount && nl <= 64) { // single-end records carry no 0x40/0x80 bit: never splitters
			SbSplitLine sl[64];
			for (int j = 0; j < nl; ++j) {
				const LineV l = read_line(V, r, j); // aligned lines keep their own coordinates and CIGAR
				sl[j].g = sb_geometry(l.cig, l.n_cig, true, l.pos + 1, l.is_rev != 0);
				sl[j].flag = l.is_rev ? 0x10 : 0; sl[j].rid = l.rid;
			}
			mask = sb_splitters(V.sb, sl, nl);
		}
		V.split_mask[r] = mask;
	}
}
struct ReadLines { const PipeView *V; int r; SSQ_HD LineV operator()(int i) const { return read_line(*V, r, i); } };
// stage 7: text of read r.  W = false: byte counts into len[*][r]; W = true: bytes at text[*] + off[*][r]
template <bool W>
SSQ_HD void body_text(const PipeView &V, int r)
{
	const ReadMeta &m = V.meta[r];
	const int nl = read_n_lines(V, r);
	LineV mh; const LineV *mate = 0;
	if (V.paired) { mh = mate_header(V, r); mate = &mh; }
	XaSrc xa; xa.tk = V.tasks + V.tk_base[r]; xa.n_tk = m.n_tasks; xa.outs = V.outs; xa.cigs = V.cigs; xa.tk_base = (int)V.tk_base[r];
	SbExtra sb; const SbExtra *sbp = 0;
	bool dup = false, disc = false; u64 smask = 0;
	if (V.sb.enabled) {
		const int u = V.paired ? r >> 1 : r;
		dup = V.dup[u] != 0; disc = V.disc[u] != 0; smask = V.split_mask[r];
		sb.or_flag = dup ? 0x400 : 0; sb.tags = false; sb.mc_cig = 0; sb.mc_n = 0; sb.mq = 0; sb.suffix = 0;
		if (V.paired && V.sb.addMateTags) {
			int mq; const SbLine mp = sb_primary(V, r ^ 1, &mq);
			sb.tags = true; sb.mc_cig = mp.cig; sb.mc_n = mp.shown ? mp.n_cig : 0; sb.mq = mq;
		}
		sbp = &sb;
	}
	Sink<W> out[3];
	for (int k = 0; k < 3; ++k) { out[k].n = 0; out[k].p = W ? V.text[k] + V.off[k][r] : 0; }
	const ReadLines ls = {&V, r};
	for (int i = 0; i < nl; ++i) {
		if (!(V.sb.enabled && V.sb.removeDups && dup)) sam_line(out[0], V.tc, r, ls, nl, i, mate, xa, sbp);
		if (V.sb.enabled) {
			if (V.sb.want_disc && disc && i == 0 && !(V.sb.excludeDups && dup)) sam_line(out[2], V.tc, r, ls, nl, i, mate, xa, sbp);
			if (V.sb.want_split && (smask >> i & 1) && !(V.sb.excludeDups && dup)) {
				SbExtra s2 = sb; s2.suffix = V.paired ? ((r & 1) ? '2' : '1') : 0;
				sam_line(out[1], V.tc, r, ls, nl, i, mate, xa, &s2);
			}
		}
	}
	if (!W) for (int k = 0; k < 3; ++k) V.len[k][r] = out[k].n;
}

// ---- BAM bodies: sizes + sort keys per line (unit = read), then the bytes (unit = sorted position) ----
struct BamCtx { LineV mh; const LineV *mate; XaSrc xa; SbExtra sb; const SbExtra *sbp; bool dup, disc; u64 smask; };
SSQ_HD void bam_ctx(const PipeView &V, int r, BamCtx &C)
{
	const ReadMeta &m = V.meta[r];
	C.mate = 0;
	if (V.paired) { C.mh = mate_header(V, r); C.mate = &C.mh; }
	C.xa.tk = V.tasks + V.tk_base[r]; C.xa.n_tk = m.n_tasks; C.xa.outs = V.outs; C.xa.cigs = V.cigs; C.xa.tk_base = (int)V.tk_base[r];
	C.sbp = 0; C.dup = C.disc = false; C.smask = 0;
	if (V.sb.enabled) {
		const int u = V.paired ? r >> 1 : r;
		C.dup = V.dup[u] != 0; C.disc = V.disc[u] != 0; C.smask = V.split_mask[r];
		C.sb.or_flag = C.dup ? 0x400 : 0; C.sb.tags = false; C.sb.mc_cig = 0; C.sb.mc_n = 0; C.sb.mq = 0; C.sb.suffix = 0;
		if (V.paired && V.sb.addMateTags) { int mq; const SbLine mp = sb_primary(V, r ^ 1, &mq); C.sb.tags = true; C.sb.mc_cig = mp.cig; C.sb.mc_n = mp.shown ? mp.n_cig : 0; C.sb.mq = mq; }
		C.sbp = &C.sb;
	}
}
SSQ_HD bool bam_member(const PipeView &V, const BamCtx &C, int k, int i)
{
	if (k == 0) return !(V.sb.enabled && V.sb.removeDups && C.dup);
	if (!V.sb.enabled || (V.sb.excludeDups && C.dup)) return false;
	return k == 2 ? (V.sb.want_disc && C.disc && i == 0) : (V.sb.want_split && (C.smask >> i & 1));
}
template <bool W>
SSQ_HD void bam_one(const PipeView &V, int r, int i, int k, const BamCtx &C, Sink<W> &out)
{
	const ReadLines ls = {&V, r};
	const int nl = read_n_lines(V, r);
	int bad = 0;
	if (k == 1) { SbExtra s2 = C.sb; s2.suffix = V.paired ? ((r & 1) ? '2' : '1') : 0; bam_record(out, V.tc, r, ls, nl, i, C.mate, C.xa, &s2, V.bam_blank_side != 0, &bad); }
	else bam_record(out, V.tc, r, ls, nl, i, C.mate, C.xa, C.sbp, k == 2 && V.bam_blank_side != 0, &bad);
	if (bad) PIPE_ERR(V, 32);
}
SSQ_HD void body_bam_size(const PipeView &V, int r)
{
	BamCtx C; bam_ctx(V, r, C);
	const int nl = read_n_lines(V, r);
	const ReadLines ls = {&V, r};
	for (int i = 0; i < nl; ++i) {
		const u64 line = V.line_base[r] + i;
		const LineV p = ls(i);
		V.bam_key[line] = bam_sort_key(patch_line(p, C.mate));
		V.line_read[line] = (u32)r;
		for (int k = 0; k < 3; ++k) {
			Sink<false> s; s.p = 0; s.n = 0;
			if (bam_member(V, C, k, i)) bam_one<false>(V, r, i, k, C, s);
			V.bam_size[k][line] = s.n;
		}
	}
}
SSQ_HD void body_bam_write(const PipeView &V, u64 sorted_pos)
{
	const u64 line = V.bam_perm[sorted_pos];
	const int r = (int)V.line_read[line], i = (int)(line - V.line_base[r]);
	BamCtx C; bam_ctx(V, r, C);
	for (int k = 0; k < 3; ++k) {
		if (!bam_member(V, C, k, i)) continue;
		Sink<true> s; s.p = V.bam[k] + V.bam_off[k][sorted_pos]; s.n = 0;
		bam_one<true>(V, r, i, k, C, s);
	}
}
