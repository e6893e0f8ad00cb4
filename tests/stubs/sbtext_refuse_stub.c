/* TEST-ONLY stand-in for libssq.so's ssq_sbtext_* entry points that refuses every chunk (SSQ_EFORMAT), so that the host fallback
 * of the `samblaster` shim's device text path (speedseq_b200/cli/samblaster_main.c built with SSQ_SB_DEVICE_TEXT) can be checked
 * against the oracle on a box without a GPU.  Linked together with dupset_stub.c by tests/test_sbtext_cpu.py; never shipped. */
#include <stdlib.h>
#include "ssq.h"
struct ssq_sbtext { ssq_dupset_t *set; uint64_t calls; };
void *ssq_host_alloc(size_t bytes) { return malloc(bytes); }
void ssq_host_free(void *p) { free(p); }
int ssq_sbtext_create(int device, const ssq_sb_opts_t *sb, const char *header, size_t header_len, ssq_sbtext_t **out)
{
	(void)sb; (void)header; (void)header_len;
	*out = (ssq_sbtext_t*)calloc(1, sizeof(**out));
	return ssq_dupset_create(device, &(*out)->set);
}
int ssq_sbtext_run(ssq_sbtext_t *s, const char *text, size_t len, int final, uint64_t max_blocks, size_t *used, ssq_sbtext_out_t *out)
{
	(void)text; (void)len; (void)final; (void)max_blocks; (void)out;
	++s->calls; *used = 0;
	return SSQ_EFORMAT;
}
ssq_dupset_t *ssq_sbtext_dupset(ssq_sbtext_t *s) { return s->set; }
void ssq_sbtext_free(ssq_sbtext_t *s) { if (s) { ssq_dupset_free(s->set); free(s); } }
