/*
 * ssqo_kseq.h — ORACLE (test infrastructure): FASTA/FASTQ tokeniser with the semantics of the
 * reference's in-tree parser speedseq/src/samtools-1.3.1/htslib-1.3.1/htslib/kseq.h:189-231
 * (name = up to first whitespace, comment = rest of header line, multi-line sequence, '+' line,
 * quality read until it is at least as long as the sequence).  gz input through zlib.
 */
#ifndef SSQO_KSEQ_H
#define SSQO_KSEQ_H
#include <stddef.h>
typedef struct { size_t l, m; char *s; } ssqo_str_t;
typedef struct ssqo_kseq_s {
	ssqo_str_t name, comment, seq, qual;
	int last_char;
	void *stream;
} ssqo_kseq_t;
ssqo_kseq_t *ssqo_kseq_open(const char *fn); /* "-" = stdin */
int ssqo_kseq_read(ssqo_kseq_t *ks);         /* >=0 sequence length; -1 EOF; -2 truncated quality */
void ssqo_kseq_close(ssqo_kseq_t *ks);
extern const unsigned char ssqo_nt4[256];
#endif
