// ssq_mem.cu — `bwa mem` for one batch through string arrays (upstream mem_process_seqs(); `$BWA mem`,
// speedseq/bin/speedseq:438,468): a convenience form of the HBM-resident pipeline in ssq_pipe.cu for callers that hold
// their reads as separate C strings.  It gathers the strings into the concatenated layout ssq_aligner_run() takes, runs one
// batch with the samblaster stage switched off, and returns the records as one malloc'd string.  The CLI shim drives a
// persistent aligner object directly (no per-batch set-up); this entry point creates and frees one per call.
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <zlib.h>
#include "ssq_host.h"
#include "ssq_samhdr.h"

extern "C" int ssq_mem_batch_sam(const ssq_index_t *idx, const ssq_opts_t *opt, int n_reads, const char *const *names, const char *const *seqs, const char *const *quals,
                                 const char *const *comments, int64_t n_processed, int paired, const ssq_pestat_t *pes0, const char *rg_id, int verbose, char **sam_out, size_t *sam_len, size_t *read_sam_off)
{
	if (!idx || !opt || n_reads < 0 || !sam_out || (n_reads && (!names || !seqs))) return SSQ_EINVAL;
	if (paired && (n_reads & 1)) { ssq_set_error("paired batch with an odd number of reads"); return SSQ_EINVAL; }
	std::string seqb, qualb, nameb, cmtb;
	std::vector<uint64_t> seq_off(n_reads + 1, 0);
	std::vector<uint32_t> name_off(n_reads + 1, 0), cmt_off(n_reads + 1, 0);
	bool has_qual = quals != 0;
	for (int i = 0; i < n_reads && has_qual; ++i) if (!quals[i]) has_qual = false;
	for (int i = 0; i < n_reads; ++i) {
		const size_t l = strlen(seqs[i]);
		seqb.append(seqs[i], l); seq_off[i + 1] = seqb.size();
		if (has_qual) { if (strlen(quals[i]) != l) { ssq_set_error("read %d: sequence and quality differ in length", i); return SSQ_EINVAL; } qualb.append(quals[i], l); }
		nameb += names[i]; name_off[i + 1] = (uint32_t)nameb.size();
		if (comments && comments[i]) cmtb += comments[i];
		cmt_off[i + 1] = (uint32_t)cmtb.size();
	}
	ssq_reads_t rd;
	memset(&rd, 0, sizeof rd);
	rd.n_reads = n_reads; rd.paired = paired; rd.seq = seqb.data(); rd.seq_off = seq_off.data(); rd.qual = has_qual ? qualb.data() : 0;
	rd.name = nameb.data(); rd.name_off = name_off.data(); rd.comment = comments ? cmtb.data() : 0; rd.comment_off = comments ? cmt_off.data() : 0; rd.n_processed = n_processed;
	ssq_aligner_t *al = 0;
	int rc = ssq_aligner_create(idx, opt, 0, rg_id, &al);
	if (rc) return rc;
	ssq_sam_t out;
	rc = ssq_aligner_run(al, &rd, pes0, verbose, &out);
	if (!rc) {
		*sam_out = (char*)malloc(out.len[0] + 1);
		if (!*sam_out) rc = SSQ_ENOMEM;
		else {
			memcpy(*sam_out, out.text[0], out.len[0]); (*sam_out)[out.len[0]] = 0;
			if (sam_len) *sam_len = out.len[0];
			if (read_sam_off) for (int i = 0; i <= n_reads; ++i) read_sam_off[i] = (size_t)out.read_off[i];
		}
	}
	ssq_aligner_free(al);
	return rc;
}

extern "C" void ssq_free(void *p) { free(p); }

// ---- BAM container (host side of f1): BGZF framing and the file header ----
// BGZF: speedseq/src/samtools-1.3.1/htslib-1.3.1/bgzf.c:45-63 — a series of gzip members of at most 64 KiB each, every member
// carrying its compressed size in a "BC" extra field, and a fixed empty member as end-of-file marker.
extern "C" int ssq_bgzf_compress(const void *in_, size_t n, int level, int with_eof, void **out, size_t *out_len)
{
	if ((!in_ && n) || !out || !out_len) return SSQ_EINVAL;
	static const unsigned char eof_blk[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
	const unsigned char *in = (const unsigned char*)in_;
	const size_t blk = 0xff00, n_blk = (n + blk - 1) / blk;
	size_t cap = n + n_blk * 64 + 64 + (level == 0 ? n_blk * 8 : 0), at = 0;
	unsigned char *o = (unsigned char*)malloc(cap);
	if (!o) return SSQ_ENOMEM;
	for (size_t b = 0; b < n_blk; ++b) {
		const size_t len = b + 1 < n_blk ? blk : n - b * blk;
		z_stream zs; memset(&zs, 0, sizeof zs);
		if (deflateInit2(&zs, level, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) { free(o); return SSQ_EINVAL; }
		if (at + 18 + deflateBound(&zs, (uLong)len) + 8 > cap) { cap = cap * 2 + deflateBound(&zs, (uLong)len) + 64; o = (unsigned char*)realloc(o, cap); }
		unsigned char *h = o + at;
		const unsigned char hdr[12] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0};
		memcpy(h, hdr, 12); h[12] = 'B'; h[13] = 'C'; h[14] = 2; h[15] = 0;
		zs.next_in = (Bytef*)(in + b * blk); zs.avail_in = (uInt)len; zs.next_out = h + 18; zs.avail_out = (uInt)(cap - at - 18 - 8);
		if (deflate(&zs, Z_FINISH) != Z_STREAM_END) { deflateEnd(&zs); free(o); ssq_set_error("deflate failed"); return SSQ_EINVAL; }
		const size_t clen = zs.total_out;
		deflateEnd(&zs);
		const unsigned bsize = (unsigned)(clen + 18 + 8 - 1);
		h[16] = (unsigned char)bsize; h[17] = (unsigned char)(bsize >> 8);
		const uLong crc = crc32(crc32(0L, 0, 0), in + b * blk, (uInt)len);
		unsigned char *t = h + 18 + clen;
		for (int k = 0; k < 4; ++k) { t[k] = (unsigned char)(crc >> (8 * k)); t[4 + k] = (unsigned char)(len >> (8 * k)); }
		at += 18 + clen + 8;
	}
	if (with_eof) { if (at + 28 > cap) o = (unsigned char*)realloc(o, at + 28); memcpy(o + at, eof_blk, 28); at += 28; }
	*out = o; *out_len = at;
	return SSQ_OK;
}

// The header text as `sambamba view -S | sambamba sort` leaves it (speedseq:440-441): "@HD VN:1.3 SO:coordinate" first (any @HD of the
// input replaced), and the tags of @SQ / @RG / @PG lines in sambamba's fixed field order (v0.5.9: SQ: SN LN AS M5 SP UR; RG: ID CN DS DT FO KS
// LB PG PI PL PU SM; PG: ID PN CL PP VN), tags it does not know after them in input order (reorder_tags, ssq_samhdr.h).  Other
// lines (@CO) pass through.
extern "C" int ssq_bam_header_text(const char *sam_header_text, int sorted, char **out)
{
	if (!out) return SSQ_EINVAL;
	std::string text;
	const char *t = sam_header_text ? sam_header_text : "";
	if (sorted) text = "@HD\tVN:1.3\tSO:coordinate\n";
	for (const char *p = t; *p;) {
		const char *e = strchr(p, '\n');
		const std::string line(p, e ? (size_t)(e - p) : strlen(p));
		p = e ? e + 1 : p + line.size();
		if (line.empty()) continue;
		if (!sorted) { text += line; text += '\n'; }
		else if (line.compare(0, 3, "@HD") != 0) reorder_tags(line, text);
	}
	*out = (char*)malloc(text.size() + 1);
	if (!*out) return SSQ_ENOMEM;
	memcpy(*out, text.c_str(), text.size() + 1);
	return SSQ_OK;
}

// "BAM\1", header text (ssq_bam_header_text), reference table — uncompressed; feed it and the records to ssq_bgzf_compress
extern "C" int ssq_bam_header(const ssq_index_t *idx, const char *sam_header_text, int sorted, void **out, size_t *out_len)
{
	if (!idx || !out || !out_len) return SSQ_EINVAL;
	char *txt = 0;
	const int rc = ssq_bam_header_text(sam_header_text, sorted, &txt);
	if (rc) return rc;
	const std::string text(txt);
	free(txt);
	std::string o("BAM\1", 4);
	auto put32 = [&](int32_t v) { char b[4] = {(char)v, (char)(v >> 8), (char)(v >> 16), (char)(v >> 24)}; o.append(b, 4); };
	put32((int32_t)text.size()); o += text;
	put32(idx->n_seqs);
	for (int i = 0; i < idx->n_seqs; ++i) { const size_t l = strlen(idx->names[i]) + 1; put32((int32_t)l); o.append(idx->names[i], l); put32(idx->ann_len[i]); }
	*out = malloc(o.size());
	if (!*out) return SSQ_ENOMEM;
	memcpy(*out, o.data(), o.size()); *out_len = o.size();
	return SSQ_OK;
}

// Merge of the coordinate-sorted runs of several batches into one sorted record stream (what `sambamba sort` does with its temporary
// files, speedseq:441).  Key = (reference id, position, strand) read from the record headers, records without a reference last; equal
// keys: the earlier run first (earlier batch = earlier input), inside a run the run's own order — i.e. a stable sort of the whole input.
extern "C" int ssq_bam_merge_runs(int n_runs, const void *const *runs, const size_t *lens, void **out, size_t *out_len)
{
	if (n_runs < 0 || (n_runs && (!runs || !lens)) || !out || !out_len) return SSQ_EINVAL;
	size_t total = 0;
	for (int r = 0; r < n_runs; ++r) total += lens[r];
	unsigned char *o = (unsigned char*)malloc(total ? total : 1);
	if (!o) return SSQ_ENOMEM;
	std::vector<size_t> at(n_runs, 0);
	auto key_of = [&](int r) -> uint64_t {
		const unsigned char *p = (const unsigned char*)runs[r] + at[r];
		int32_t ref, pos; uint16_t flag;
		memcpy(&ref, p + 4, 4); memcpy(&pos, p + 8, 4); memcpy(&flag, p + 4 + 14, 2); // block_size | refID pos l_read_name mapq bin n_cigar flag ...
		return ref < 0 ? ~0ull : ((uint64_t)(uint32_t)ref << 34 | (uint64_t)(pos + 1) << 1 | (uint64_t)((flag >> 4) & 1));
	};
	size_t w = 0;
	for (;;) { // n_runs is small (batches of one run): a linear scan for the minimum keeps the earlier run on ties
		int best = -1; uint64_t bk = 0;
		for (int r = 0; r < n_runs; ++r) {
			if (at[r] + 4 > lens[r]) continue;
			const uint64_t k = key_of(r);
			if (best < 0 || k < bk) { best = r; bk = k; }
		}
		if (best < 0) break;
		const unsigned char *p = (const unsigned char*)runs[best] + at[best];
		int32_t bs; memcpy(&bs, p, 4);
		if (bs < 32 || at[best] + 4 + (size_t)bs > lens[best]) { free(o); ssq_set_error("ssq_bam_merge_runs: run %d is not a sequence of BAM records", best); return SSQ_EINVAL; }
		memcpy(o + w, p, 4 + (size_t)bs); w += 4 + (size_t)bs; at[best] += 4 + (size_t)bs;
	}
	*out = o; *out_len = w;
	return SSQ_OK;
}
