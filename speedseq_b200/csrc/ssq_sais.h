// ssq_sais.h — suffix array by induced sorting (SA-IS: Nong, Zhang, Chan, "Two efficient algorithms for linear time suffix array
// construction", 2011), host code.  `ssq_index_build` uses it for references whose 2 x l_pac + 1 suffixes exceed what the GPU
// prefix-doubling sort of this build holds (2^31 - 2): `$BWA index $REF` on a whole genome, speedseq/bin/speedseq:386-391
// (SURVEY §8 f3: "GPU suffix sort optional").  Upstream bwa switches to its own incremental BWT construction above 50 Mbp; the
// index files do not record how the suffix array was obtained.
//
// ssq_sais(s, SA, n, K): s[0..n) over the alphabet [0, K), s[n-1] = 0 the unique smallest symbol (sentinel); SA[0..n) receives
// the suffix array (SA[0] = n - 1).  `SA` is anything pointer-like over signed integers wide enough for n: int32_t*, int64_t*, or
// ssq_p40 — 40-bit entries (5 bytes per suffix: a whole human genome's 6.2 G suffixes in 31 GB instead of 50).  Working space
// beyond SA: n bits of suffix types and a bucket array of K entries per level; the reduced string of a recursion level and its
// suffix array live inside SA, as in the original formulation.
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

// pointer-like view of 40-bit entries; all ones reads as -1 (the "empty" mark of the algorithm); the buffer needs 3 bytes of slack
struct ssq_r40 {
	uint8_t *p;
	operator int64_t() const { uint64_t x; memcpy(&x, p, 8); x &= 0xffffffffffull; return x == 0xffffffffffull ? -1 : (int64_t)x; }
	ssq_r40 &operator=(int64_t v) { const uint64_t x = (uint64_t)v; memcpy(p, &x, 5); return *this; }
	ssq_r40 &operator=(const ssq_r40 &o) { return *this = (int64_t)o; }
};
struct ssq_p40 {
	uint8_t *p;
	ssq_r40 operator[](int64_t i) const { ssq_r40 r; r.p = p + 5 * i; return r; }
	ssq_p40 operator+(int64_t d) const { ssq_p40 q; q.p = p + 5 * d; return q; }
};

namespace ssq_sais_detail {

typedef int64_t I; // index arithmetic; the storage type is the SA view's business

template <class TXT>
static void bucket_bounds(TXT s, std::vector<I> &bkt, I n, I K, bool end)
{
	for (I i = 0; i < K; ++i) bkt[(size_t)i] = 0;
	for (I i = 0; i < n; ++i) ++bkt[(size_t)(I)s[i]];
	I sum = 0;
	for (I i = 0; i < K; ++i) { sum += bkt[(size_t)i]; bkt[(size_t)i] = end ? sum : sum - bkt[(size_t)i]; }
}

struct TypeBits { // bit i set: suffix i is S-type
	std::vector<uint64_t> w;
	explicit TypeBits(size_t n) : w((n + 63) / 64, 0) {}
	bool get(size_t i) const { return (w[i >> 6] >> (i & 63)) & 1; }
	void set(size_t i, bool v) { if (v) w[i >> 6] |= 1ull << (i & 63); else w[i >> 6] &= ~(1ull << (i & 63)); }
};
static inline bool is_lms(const TypeBits &t, I i) { return i > 0 && t.get((size_t)i) && !t.get((size_t)i - 1); }

template <class TXT, class SAP>
static void induce_l(const TypeBits &t, SAP SA, TXT s, std::vector<I> &bkt, I n, I K)
{
	bucket_bounds(s, bkt, n, K, false);
	for (I i = 0; i < n; ++i) {
		const I v = SA[i], j = v - 1;
		if (v > 0 && !t.get((size_t)j)) SA[bkt[(size_t)(I)s[j]]++] = j;
	}
}
template <class TXT, class SAP>
static void induce_s(const TypeBits &t, SAP SA, TXT s, std::vector<I> &bkt, I n, I K)
{
	bucket_bounds(s, bkt, n, K, true);
	for (I i = n - 1; i >= 0; --i) {
		const I v = SA[i], j = v - 1;
		if (v > 0 && t.get((size_t)j)) SA[--bkt[(size_t)(I)s[j]]] = j;
	}
}

template <class TXT, class SAP>
static void sais_rec(TXT s, SAP SA, I n, I K)
{
	TypeBits t((size_t)n);
	t.set((size_t)n - 1, true);
	if (n >= 2) t.set((size_t)n - 2, false);
	for (I i = n - 3; i >= 0; --i) { const I a = s[i], b = s[i + 1]; t.set((size_t)i, a < b || (a == b && t.get((size_t)i + 1))); }
	std::vector<I> bkt((size_t)K);
	// stage 1: sort the LMS substrings by one round of induced sorting
	bucket_bounds(s, bkt, n, K, true);
	for (I i = 0; i < n; ++i) SA[i] = -1;
	for (I i = 1; i < n; ++i) if (is_lms(t, i)) SA[--bkt[(size_t)(I)s[i]]] = i;
	induce_l(t, SA, s, bkt, n, K);
	induce_s(t, SA, s, bkt, n, K);
	// the sorted LMS suffixes to the front
	I n1 = 0;
	for (I i = 0; i < n; ++i) { const I v = SA[i]; if (is_lms(t, v)) SA[n1++] = v; }
	// names: equal LMS substrings get equal names; stored at SA[n1 + pos / 2]
	for (I i = n1; i < n; ++i) SA[i] = -1;
	I name = 0, prev = -1;
	for (I i = 0; i < n1; ++i) {
		const I pos = SA[i];
		bool diff = false;
		for (I d = 0; d < n; ++d) {
			if (prev == -1 || (I)s[pos + d] != (I)s[prev + d] || t.get((size_t)(pos + d)) != t.get((size_t)(prev + d))) { diff = true; break; }
			if (d > 0 && (is_lms(t, pos + d) || is_lms(t, prev + d))) break;
		}
		if (diff) { ++name; prev = pos; }
		SA[n1 + pos / 2] = name - 1;
	}
	for (I i = n - 1, j = n - 1; i >= n1; --i) { const I v = SA[i]; if (v >= 0) SA[j--] = v; }
	// stage 2: the order of the LMS suffixes = suffix array of the reduced string
	SAP SA1 = SA, s1 = SA + (n - n1);
	if (name < n1) sais_rec<SAP, SAP>(s1, SA1, n1, name);
	else for (I i = 0; i < n1; ++i) SA1[(I)s1[i]] = i;
	// stage 3: induce the whole suffix array from the sorted LMS suffixes
	bucket_bounds(s, bkt, n, K, true);
	for (I i = 1, j = 0; i < n; ++i) if (is_lms(t, i)) s1[j++] = i; // positions of the LMS suffixes in text order
	for (I i = 0; i < n1; ++i) { const I v = s1[(I)SA1[i]]; SA1[i] = v; }
	for (I i = n1; i < n; ++i) SA[i] = -1;
	for (I i = n1 - 1; i >= 0; --i) {
		const I j = SA[i];
		SA[i] = -1;
		SA[--bkt[(size_t)(I)s[j]]] = j;
	}
	induce_l(t, SA, s, bkt, n, K);
	induce_s(t, SA, s, bkt, n, K);
}

} // namespace ssq_sais_detail

template <class SAP>
static void ssq_sais(const uint8_t *s, SAP SA, int64_t n, int64_t K)
{
	if (n <= 0) return;
	if (n == 1) { SA[0] = 0; return; }
	ssq_sais_detail::sais_rec<const uint8_t*, SAP>(s, SA, n, K);
}
