/*
 * oracle/ref_harness.c — TEST INFRASTRUCTURE ONLY (never linked into libvdl2gpu.so).
 *
 * Driver for the UNMODIFIED reference hot path.  The reference translation units
 *   src/demod.c src/chebyshev.c src/rs.c src/bitstream.c src/decode.c src/crc.c
 *   src/libfec/init_rs_char.c src/libfec/decode_rs_char.c
 * are compiled where they lie under /root/reference (see oracle/Makefile) against the
 * stand-in headers in oracle/ref_shim/, and linked with this file, which supplies what
 * the rest of dumpvdl2 would have supplied:
 *   - the globals `Config`, `do_exit`, `demods_ready`, `samples_ready`   (reference src/dumpvdl2.c:65-67)
 *   - `xcalloc`, `octet_string_new`                                       (reference src/util.c:32,145)
 *   - the GAsyncQueue calls; push == capture (metadata, frame) per channel (reference src/decode.c:165-171)
 *   - the thread/barrier protocol of start_demod_threads/process_iq_file   (reference src/dumpvdl2.c:117-135,323-358,1170)
 * Nothing here restates reference arithmetic: every sample goes through the reference's own
 * process_buf_uchar/process_buf_short -> process_samples -> demod -> decode_vdl2_burst.
 *
 * Usage: vdl2_ref --fmt u8|s16 --oversample N --centerfreq HZ --freqs f0,f1,... [--chunk BYTES]
 *                 [--max-ppm X] [--loop N] [--quiet] [--pin] [--debug MASK] FILE
 *        --pin: channel thread i is bound to CPU i mod (online CPUs), the producer to the last CPU (timing runs)
 * Output (stdout): one line per pushed frame, sorted by (channel, push order):
 *   FRAME ch=I freq=F idx=K len=L synd=W datalen=D fec=C pwr=%.9g nf=%.9g ppm=%.9g hex=...
 * and a final  STATS ...  line with wall time of the sample loop.
 */
#define _GNU_SOURCE
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <time.h>
#include <pthread.h>
#include <sched.h>
#include <unistd.h>
#include <glib.h>
#include <libacars/libacars.h>
#include <libacars/list.h>
#include <libacars/reassembly.h>
#include "dumpvdl2.h"
#include "decode.h"
#include "avlc.h"
#include "output-common.h"
#include "reassembly.h"

/* ---- globals the hot path expects from dumpvdl2.c ---- */
dumpvdl2_config_t Config;
int do_exit = 0;
pthread_barrier_t demods_ready, samples_ready;

/* ---- util.c stand-ins ---- */
void *xcalloc(size_t nmemb, size_t size, char const *file, int line, char const *func) {
	void *p = calloc(nmemb ? nmemb : 1, size ? size : 1);
	if(p == NULL) {
		fprintf(stderr, "%s:%d %s: calloc failed\n", file, line, func);
		_exit(1);
	}
	return p;
}
octet_string_t *octet_string_new(void *buf, size_t len) {
	octet_string_t *o = calloc(1, sizeof(*o));
	o->buf = buf;
	o->len = len;
	return o;
}
void octet_string_destroy(octet_string_t *o) {
	if(o) { free(o->buf); free(o); }
}

/* ---- never reached on the demod side; present to satisfy the linker (decode.c:386-527) ---- */
la_proto_node *avlc_parse(avlc_frame_qentry_t *q, uint32_t *t, reasm_contexts *r) { (void)q; (void)t; (void)r; return NULL; }
la_list *la_list_next(la_list const *l) { return l ? l->next : NULL; }
void la_list_foreach(la_list *l, void (*cb)(void *, void *), void *ctx) { (void)l; (void)cb; (void)ctx; }
void la_proto_tree_destroy(la_proto_node *root) { (void)root; }
la_reasm_ctx *la_reasm_ctx_new(void) { return NULL; }
reasm_ctx *reasm_ctx_new() { return NULL; }
output_qentry_t *output_qentry_copy(output_qentry_t const *q) { (void)q; return NULL; }

/* ---- frame capture ---- */
typedef struct captured {
	vdl2_msg_metadata md;
	uint8_t *buf;
	size_t len;
	struct captured *next;
} captured_t;

typedef struct {
	captured_t *head, *tail;
	size_t count;
} chan_capture_t;

static chan_capture_t *captures;
static int num_channels;
static int keep_frames = 1;
static __thread int tl_chan = -1;
static uint32_t *chan_freqs;
static pthread_mutex_t capture_lock = PTHREAD_MUTEX_INITIALIZER;

struct shim_async_queue { int unused; };
static struct shim_async_queue the_queue;
GAsyncQueue *g_async_queue_new(void) { return &the_queue; }
int g_async_queue_length(GAsyncQueue *q) { (void)q; return 0; }
void *g_async_queue_pop(GAsyncQueue *q) { (void)q; return NULL; }

void g_async_queue_push(GAsyncQueue *q, void *item) {
	(void)q;
	avlc_frame_qentry_t *e = item;
	if(tl_chan < 0 || tl_chan >= num_channels) {
		fprintf(stderr, "frame pushed from a non-channel thread\n");
		_exit(4);
	}
	/* The reference pushes from the channel's own thread.  A drop-in demodulator may push every channel's
	 * frames from one thread: then the channel is recovered from the metadata (first channel on that frequency). */
	int chan = tl_chan;
	if(chan_freqs[chan] != e->metadata->freq) {
		for(chan = 0; chan < num_channels && chan_freqs[chan] != e->metadata->freq; chan++) ;
		if(chan == num_channels) { fprintf(stderr, "frame for an unknown frequency\n"); _exit(4); }
	}
	pthread_mutex_lock(&capture_lock);
	chan_capture_t *cc = &captures[chan];
	cc->count++;
	if(keep_frames) {
		captured_t *c = calloc(1, sizeof(*c));
		c->md = *e->metadata;
		c->len = e->frame->len;
		c->buf = malloc(c->len ? c->len : 1);
		memcpy(c->buf, e->frame->buf, c->len);
		if(cc->tail) cc->tail->next = c; else cc->head = c;
		cc->tail = c;
	}
	pthread_mutex_unlock(&capture_lock);
	octet_string_destroy(e->frame);
	free(e->metadata);
	free(e);
}

/* ---- channel threads ---- */
typedef struct { int idx; vdl2_channel_t *v; } thr_arg_t;

static void *chan_thread(void *arg) {
	thr_arg_t *a = arg;
	tl_chan = a->idx;
	return process_samples(a->v);   /* never returns */
}

/* one FRAME line per captured frame, by channel in push order; returns the number of frames */
static size_t print_captures(void) {
	size_t nframes = 0;
	for(int i = 0; i < num_channels; i++) {
		nframes += captures[i].count;
		for(captured_t *c = captures[i].head; c; c = c->next) {
			printf("FRAME ch=%d freq=%u idx=%d len=%zu synd=%u datalen=%u fec=%d pwr=%.9g nf=%.9g ppm=%.9g hex=",
					i, c->md.freq, c->md.idx, c->len, c->md.synd_weight, c->md.datalen_octets,
					c->md.num_fec_corrections, c->md.frame_pwr_dbfs, c->md.nf_pwr_dbfs, c->md.ppm_error);
			for(size_t k = 0; k < c->len; k++) printf("%02x", c->buf[k]);
			printf("\n");
		}
	}
	return nframes;
}

static double now_s(void) {
	struct timespec ts;
	clock_gettime(CLOCK_MONOTONIC, &ts);
	return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

#ifndef REF_HARNESS_NO_MAIN
int main(int argc, char **argv) {
	char const *fmt = "u8", *freqs_s = NULL, *file = NULL;
	uint32_t oversample = 10, centerfreq = 0, chunk = FILE_BUFSIZE;
	int loops = 1, quiet = 0, pin = 0;
	memset(&Config, 0, sizeof(Config));
	for(int i = 1; i < argc; i++) {
		if(!strcmp(argv[i], "--fmt") && i+1 < argc) fmt = argv[++i];
		else if(!strcmp(argv[i], "--oversample") && i+1 < argc) oversample = strtoul(argv[++i], NULL, 10);
		else if(!strcmp(argv[i], "--centerfreq") && i+1 < argc) centerfreq = strtoul(argv[++i], NULL, 10);
		else if(!strcmp(argv[i], "--freqs") && i+1 < argc) freqs_s = argv[++i];
		else if(!strcmp(argv[i], "--chunk") && i+1 < argc) chunk = strtoul(argv[++i], NULL, 10);
		else if(!strcmp(argv[i], "--max-ppm") && i+1 < argc) Config.max_ppm = strtof(argv[++i], NULL);
		else if(!strcmp(argv[i], "--loop") && i+1 < argc) loops = atoi(argv[++i]);
		else if(!strcmp(argv[i], "--quiet")) quiet = 1;
		else if(!strcmp(argv[i], "--pin")) pin = 1;
		else if(!strcmp(argv[i], "--debug") && i+1 < argc) {
#ifdef DEBUG
			Config.debug_filter = strtoul(argv[++i], NULL, 0);
#else
			++i;
#endif
		}
		else if(argv[i][0] != '-') file = argv[i];
		else { fprintf(stderr, "unknown option %s\n", argv[i]); return 2; }
	}
	if(!file || !freqs_s) { fprintf(stderr, "need --freqs and FILE\n"); return 2; }
	int is_s16 = !strcmp(fmt, "s16");
	keep_frames = !quiet;

	/* parse frequency list */
	uint32_t *freqs = NULL;
	{
		char *dup = strdup(freqs_s), *save = NULL;
		for(char *t = strtok_r(dup, ",", &save); t; t = strtok_r(NULL, ",", &save)) {
			freqs = realloc(freqs, (num_channels + 1) * sizeof(uint32_t));
			freqs[num_channels++] = strtoul(t, NULL, 10);
		}
		free(dup);
	}
	if(centerfreq == 0) centerfreq = freqs[0];
	chan_freqs = freqs;
	uint32_t sample_rate = SYMBOL_RATE * SPS * oversample;       /* reference src/dumpvdl2.c:1073 */

	/* load the whole input into RAM */
	FILE *f = fopen(file, "rb");
	if(!f) { perror(file); return 2; }
	fseek(f, 0, SEEK_END);
	long fsize = ftell(f);
	fseek(f, 0, SEEK_SET);
	unsigned char *data = malloc(fsize ? fsize : 1);
	if(fread(data, 1, fsize, f) != (size_t)fsize) { perror("fread"); return 2; }
	fclose(f);

	/* init order mirrors reference src/dumpvdl2.c:1086-1153 */
	captures = calloc(num_channels, sizeof(*captures));
	vdl2_channel_t **chans = calloc(num_channels, sizeof(*chans));
	for(int i = 0; i < num_channels; i++)
		chans[i] = vdl2_channel_init(centerfreq, freqs[i], sample_rate, oversample);
	if(rs_init() < 0) { fprintf(stderr, "rs_init failed\n"); return 3; }
	avlc_decoder_init();
	sincosf_lut_init();
	input_lpf_init(sample_rate);
	demod_sync_init();
	process_buf_uchar_init();
	sbuf = calloc(chunk, sizeof(float));
	pthread_barrier_init(&demods_ready, NULL, num_channels + 1);
	pthread_barrier_init(&samples_ready, NULL, num_channels + 1);
	thr_arg_t *targs = calloc(num_channels, sizeof(*targs));
	for(int i = 0; i < num_channels; i++) {
		targs[i].idx = i;
		targs[i].v = chans[i];
		pthread_create(&chans[i]->demod_thread, NULL, chan_thread, &targs[i]);
	}
	if(pin) {
		/* the CPUs this process may use, in order; channel i -> the (i mod n-1)-th of them, producer -> the last */
		cpu_set_t all;
		CPU_ZERO(&all);
		sched_getaffinity(0, sizeof(all), &all);
		int cpus[CPU_SETSIZE], ncpu = 0;
		for(int c = 0; c < CPU_SETSIZE; c++) if(CPU_ISSET(c, &all)) cpus[ncpu++] = c;
		if(ncpu > 1) {
			for(int i = 0; i < num_channels; i++) {
				cpu_set_t one;
				CPU_ZERO(&one);
				CPU_SET(cpus[i % (ncpu - 1)], &one);
				pthread_setaffinity_np(chans[i]->demod_thread, sizeof(one), &one);
			}
			cpu_set_t one;
			CPU_ZERO(&one);
			CPU_SET(cpus[ncpu - 1], &one);
			pthread_setaffinity_np(pthread_self(), sizeof(one), &one);
		}
	}

	/* feed chunks like process_iq_file (reference src/dumpvdl2.c:353-356); the file is NOT
	 * header-skipped, exactly as in the reference */
	double t0 = now_s();
	uint64_t total_bytes = 0;
	for(int l = 0; l < loops; l++) {
		for(long off = 0; off < fsize; off += chunk) {
			uint32_t len = (uint32_t)((fsize - off) < (long)chunk ? (fsize - off) : (long)chunk);
			if(is_s16) process_buf_short(data + off, len, NULL);
			else process_buf_uchar(data + off, len, NULL);
			total_bytes += len;
		}
	}
	pthread_barrier_wait(&demods_ready);     /* drain: reference src/dumpvdl2.c:1170 */
	double t1 = now_s();

	size_t nframes = print_captures();
	uint64_t iq_samples = total_bytes / (is_s16 ? 4 : 2);
	printf("STATS channels=%d iq_samples=%llu frames=%zu wall_s=%.6f ch_msamples_per_s=%.3f\n",
			num_channels, (unsigned long long)iq_samples, nframes, t1 - t0,
			(double)num_channels * (double)iq_samples / (t1 - t0) / 1e6);
	fflush(stdout);
	_exit(0);   /* channel threads are parked on the barrier; no join (same as the reference's shutdown) */
}
#endif
