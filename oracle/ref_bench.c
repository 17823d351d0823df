/*
 * oracle/ref_bench.c -- TEST/BENCH INFRASTRUCTURE ONLY (never linked into the product).
 *
 * A pthread harness around a decoder of the 15-function ABI: the UNMODIFIED reference decoder
 * (reference src/wasm/mpeg1.c + buffer.c, compiled in place by oracle/Makefile into
 * oracle/_ref/libjsmpeg_ref.so) and, built with ORACLE_ABI, the oracle (oracle/liboracle.so), so that
 * the checker and the hash also exist where the reference tree is absent.  It only
 * uses the reference's public 15-function ABI (reference src/wasm/mpeg1.h:10-25), exactly the
 * way the reference's own glue does (src/mpeg1-wasm.js:52-70 write, :103 decode): one decoder
 * per elementary stream, whole stream written once (EXPAND mode), then decode() until it
 * returns false.  This is the `cpu_baseline` / `--impl reference` arm of bench.py, and (through
 * ref_picture_hashes) the checker bench.py and the GPU tests hold the CUDA output against.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#ifdef ORACLE_ABI
#include "../include/jsmpeg_b200.h"
#else
#include "mpeg1.h"
#endif

typedef struct {
	const uint8_t *const *es;
	const unsigned *es_len;
	int n_clips, first, stride, loops;
	long frames;
	uint64_t checksum;
	pthread_barrier_t *start, *stop;
} job_t;

static uint64_t fnv1a(uint64_t h, const uint8_t *p, size_t n) {
	for (size_t i = 0; i < n; i++) { h ^= p[i]; h *= 1099511628211ULL; }
	return h;
}

static mpeg1_decoder_t *open_clip(const uint8_t *es, unsigned len) {
	mpeg1_decoder_t *d = mpeg1_decoder_create(len + 16, BIT_BUFFER_MODE_EXPAND);
	memcpy(mpeg1_decoder_get_write_ptr(d, len), es, len);
	mpeg1_decoder_did_write(d, len);
	return d;
}

static void *worker(void *arg) {
	job_t *j = (job_t *)arg;
	/* every decoder this thread will use is created and written BEFORE the clock starts */
	int mine = 0;
	for (int c = j->first; c < j->n_clips; c += j->stride) mine++;
	const int total = mine * j->loops;
	mpeg1_decoder_t **dec = (mpeg1_decoder_t **)calloc(total ? total : 1, sizeof(*dec));
	int k = 0;
	for (int l = 0; l < j->loops; l++)
		for (int c = j->first; c < j->n_clips; c += j->stride) dec[k++] = open_clip(j->es[c], j->es_len[c]);
	pthread_barrier_wait(j->start);
	for (k = 0; k < total; k++) {
		while (mpeg1_decoder_decode(dec[k])) j->frames++;
		/* touch the last picture so the decode cannot be optimised away */
		if (mpeg1_decoder_has_sequence_header(dec[k])) j->checksum = fnv1a(j->checksum, (const uint8_t *)mpeg1_decoder_get_y_ptr(dec[k]), 64);
	}
	pthread_barrier_wait(j->stop);
	for (k = 0; k < total; k++) mpeg1_decoder_destroy(dec[k]);
	free(dec);
	return 0;
}

/* Decode n_clips elementary streams `loops` times on `threads` host threads (clip c is handled
 * by thread c % threads).  Returns the number of pictures decode() reported; *seconds gets the
 * wall time of the decode() loops alone: decoder creation, the write of the stream and the
 * destruction happen outside the timed region (two barriers). */
long ref_bench_run(const uint8_t *const *es, const unsigned *es_len, int n_clips,
                   int threads, int loops, double *seconds) {
	if (threads < 1) threads = 1;
	pthread_t *tid = (pthread_t *)calloc(threads, sizeof(pthread_t));
	job_t *jobs = (job_t *)calloc(threads, sizeof(job_t));
	pthread_barrier_t start, stop;
	pthread_barrier_init(&start, 0, threads + 1);
	pthread_barrier_init(&stop, 0, threads + 1);
	struct timespec t0, t1;
	for (int t = 0; t < threads; t++) {
		jobs[t].es = es; jobs[t].es_len = es_len; jobs[t].n_clips = n_clips;
		jobs[t].first = t; jobs[t].stride = threads; jobs[t].loops = loops;
		jobs[t].checksum = 1469598103934665603ULL;
		jobs[t].start = &start; jobs[t].stop = &stop;
		pthread_create(&tid[t], 0, worker, &jobs[t]);
	}
	pthread_barrier_wait(&start);
	clock_gettime(CLOCK_MONOTONIC, &t0);
	pthread_barrier_wait(&stop);
	clock_gettime(CLOCK_MONOTONIC, &t1);
	long frames = 0;
	for (int t = 0; t < threads; t++) { pthread_join(tid[t], 0); frames += jobs[t].frames; }
	if (seconds) *seconds = (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
	pthread_barrier_destroy(&start);
	pthread_barrier_destroy(&stop);
	free(tid); free(jobs);
	return frames;
}

/* Checker for the GPU arm (tests, bench.py's `verified`): decodes one elementary stream with the
 * reference and writes, per decode() == true, the FNV-1a 64 hash of the picture the reference would
 * hand to its renderer (get_y_ptr | get_cr_ptr | get_cb_ptr, coded size) into hashes[0 .. max).
 * Returns the number of pictures. */
long ref_picture_hashes(const uint8_t *es, unsigned es_len, uint64_t *hashes, long max) {
	mpeg1_decoder_t *d = open_clip(es, es_len);
	long n = 0;
	while (mpeg1_decoder_decode(d)) {
		if (n < max) {
			const size_t ysz = (size_t)mpeg1_decoder_get_coded_size(d);
			uint64_t h = 1469598103934665603ULL;
			h = fnv1a(h, (const uint8_t *)mpeg1_decoder_get_y_ptr(d), ysz);
			h = fnv1a(h, (const uint8_t *)mpeg1_decoder_get_cr_ptr(d), ysz >> 2);
			h = fnv1a(h, (const uint8_t *)mpeg1_decoder_get_cb_ptr(d), ysz >> 2);
			hashes[n] = h;
		}
		n++;
	}
	mpeg1_decoder_destroy(d);
	return n;
}

/* FNV-1a 64 continuation over caller memory: lets the checker hash the GPU arm's planes with the
 * very function that hashed the reference's (the hash is serial; Python would take seconds per picture). */
uint64_t ref_hash_bytes(uint64_t h, const uint8_t *p, size_t n) { return fnv1a(h, p, n); }
