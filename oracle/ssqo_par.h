/* ssqo_par.h — ORACLE (test infrastructure): minimal pthread parallel-for (dynamic chunks of 16),
 * the stand-in for bwa's kt_for worker pool (`bwa mem -t N`, speedseq/bin/speedseq:438). */
#ifndef SSQO_PAR_H
#define SSQO_PAR_H
#include <pthread.h>
#include <stdlib.h>
typedef struct { void (*fn)(void*, long, int); void *data; long n; volatile long next; } ssqo_par_t;
typedef struct { ssqo_par_t *p; int tid; } ssqo_par_arg_t;
static void *ssqo_par_worker(void *a_)
{
	ssqo_par_arg_t *a = (ssqo_par_arg_t*)a_;
	for (;;) {
		long i = __sync_fetch_and_add(&a->p->next, 16), e;
		if (i >= a->p->n) break;
		e = i + 16 < a->p->n ? i + 16 : a->p->n;
		for (; i < e; ++i) a->p->fn(a->p->data, i, a->tid);
	}
	return 0;
}
static void ssqo_parallel_for(int n_threads, long n, void (*fn)(void*, long, int), void *data)
{
	ssqo_par_t p;
	p.fn = fn; p.data = data; p.n = n; p.next = 0;
	if (n_threads <= 1) { long i; for (i = 0; i < n; ++i) fn(data, i, 0); return; }
	{
		pthread_t *tid = (pthread_t*)malloc(sizeof(pthread_t) * n_threads);
		ssqo_par_arg_t *arg = (ssqo_par_arg_t*)malloc(sizeof(ssqo_par_arg_t) * n_threads);
		int i;
		for (i = 0; i < n_threads; ++i) { arg[i].p = &p; arg[i].tid = i; pthread_create(&tid[i], 0, ssqo_par_worker, &arg[i]); }
		for (i = 0; i < n_threads; ++i) pthread_join(tid[i], 0);
		free(tid); free(arg);
	}
}
#endif
