/*
 * jpegqs.c - the `jpegqs` command line tool on top of the CUDA (sm_90a) back end.
 *
 * Same command line surface as the reference tool (reference quantsmooth.c:288-393):
 *   jpegqs [options] input.jpg output.jpg        ("-" = stdin / stdout)
 *     -q, --quality n    0..6, default 3 (mapped to flags exactly like quantsmooth.c:380-393)
 *     -n, --niter n      number of iterations (default 3)
 *     -t, --threads n    worker threads of the JPEG reader's and writer's entropy coding (the
 *                        reference: OpenMP threads of the smoothing loop, which runs on the GPU here)
 *     -o, --optimize     optimal Huffman tables in the output
 *     -v, --verbose n    codec diagnostics
 *     -i, --info n       info bit mask (JPEGQS_INFO_*), default 15
 *     -p, --cpu n        CUDA device ordinal + 1 (0 = current device); the reference's SIMD cap
 *     -f, --flags n      raw JPEGQS_* flag bits instead of -q
 *     -c, --copy n       0 = no markers, 1 = comments, 2 = comments + APPn (default)
 *     --batch            (extension) any number of "input output" pairs follow: one process, CUDA
 *                        start-up paid once (it is 1-2 s in a fresh process, 100x the smoothing
 *                        of an 8K image); reading, smoothing and writing of successive pairs
 *                        overlap (JPEGQS_NO_PIPELINE=1: one pair after the other); exit status =
 *                        the worst of the pairs
 *     --ppm              (extension) write the decoded RGB image as binary PPM/PGM instead of a
 *                        JPEG: the device-side equivalent of the reference's example.c
 *                        (JPEG -> pixels through jpegqs_start_decompress)
 * The flow is the reference's (quantsmooth.c:494-596): read coefficients, do_quantsmooth,
 * write coefficients + copied markers.  libjpeg is replaced by jpegcoef.c because its headers
 * are not available in this build image.  Exit code: 0 ok, 1 usage / I/O / codec error,
 * 2 when the input had recoverable damage (the reference: libjpeg warnings, quantsmooth.c:626)
 * or the CUDA back end failed (negative do_quantsmooth return).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <jpeglib.h>
#include "libjpegqs.h"
#include "jpegcoef.h"
#ifndef JPEGQS_NO_CUDA_RENDER      /* the reference-linked test build (oracle/Makefile) has no CUDA back end */
#include "jpegqs_cuda.h"
#include <pthread.h>
static void *warmup_thread(void *arg) { jpegqs_warmup(*(int*)arg); return NULL; }
#endif
#include <sys/time.h>
#ifdef __GLIBC__
#include <malloc.h>
#endif
static double now_ms(void) { struct timeval tv; gettimeofday(&tv, NULL); return tv.tv_sec * 1e3 + tv.tv_usec * 1e-3; }

static unsigned char *load_all(FILE *f, size_t *len) {
	size_t cap = 1 << 20, n = 0, r; unsigned char *p = (unsigned char*)malloc(cap);
	if (!p) return NULL;
	while ((r = fread(p + n, 1, cap - n, f)) > 0) {
		n += r;
		if (n == cap) { unsigned char *q = (unsigned char*)realloc(p, cap *= 2); if (!q) { free(p); return NULL; } p = q; }
	}
	*len = n;
	return p;
}

static int usage(const char *prog) {
	fprintf(stderr,
		"jpegqs (CUDA sm_90a back end) version " JPEGQS_VERSION "\n"
		"Usage:\n  %s [options] input.jpg output.jpg\n\nOptions:\n"
		"  -q, --quality n   Quality setting (0-6, default is 3)\n"
		"  -n, --niter n     Number of iterations (default is 3)\n"
		"  -t, --threads n   Worker threads of the JPEG reader and writer (the reference: OpenMP threads)\n"
		"  -o, --optimize    Optimize Huffman table\n"
		"  -v, --verbose n   Print codec debug messages\n"
		"  -i, --info n      Print quantsmooth debug messages (default is 15)\n"
		"  -p, --cpu n       CUDA device ordinal + 1 (0 = current device)\n"
		"  -f, --flags n     Raw flag bits\n"
		"  -c, --copy n      Markers to copy: 0 none, 1 comments, 2 all (default)\n"
		"      --batch       Process several \"input output\" pairs in one process\n"
		"      --ppm         Write the decoded image (PPM/PGM) instead of a JPEG\n", prog);
	return 1;
}

/* One "input output" pair moves through three stages: read + Huffman-decode, do_quantsmooth,
 * encode + write.  A single pair runs them in a row; --batch runs them as a pipeline (a reader
 * thread, the calling thread for the device work, a writer thread), so that with many files the
 * process moves at the pace of the slowest stage instead of their sum.
 * The device route (jpegqs_transcode): when the file allows it, the reader only loads the bytes, the
 * middle stage decodes, smooths and encodes on the device and the writer only writes the result -
 * the same bytes, exit status and messages as the host codec around do_quantsmooth. */
typedef struct {
	const char *in_name, *out_name;
	int state;                           /* stages completed: 0 none, 1 read, 2 smoothed, 3 written */
	int rc;                              /* exit status of this pair so far (non-zero: later stages are skipped) */
	int have_im;
	jq_image im;
	unsigned char *data; size_t len;     /* device route: the input file, then (out) the output file */
	unsigned char *out; size_t outlen;
	size_t held;                         /* --batch: bytes counted against the readers' look-ahead */
	double t_read, t_smooth, t_write;    /* stage durations, ms */
} qs_job;

typedef struct {
	const char *prog;
	jpegqs_control_t opts;
	int copy, optimize, verbose, ppm, cpu;
	const char *host_only;               /* why no pair takes the device route, NULL if pairs may */
	int trace;                           /* JPEGQS_CODEC_TRACE: print the route of every pair */
} qs_cfg;

/* the reader's part of the host route: Huffman-decode the file (consumes data) */
static void job_decode(const qs_cfg *g, qs_job *j, unsigned char *data, size_t len, int header_line) {
	char err[256];
	if (jq_read(data, len, g->copy, &j->im, err)) { fprintf(stderr, "%s: %s\n", g->prog, err); free(data); j->rc = 1; return; }
	free(data);
	j->have_im = 1;
	if (g->verbose && header_line)
		fprintf(stderr, "%s: %ux%u, %d component(s), %s, restart interval %d\n", j->in_name, j->im.cinfo.image_width,
				j->im.cinfo.image_height, j->im.cinfo.num_components, j->im.progressive ? "progressive" : "sequential",
				j->im.restart_interval);
}

/* host_wait (may be NULL): called before a host-route pair is Huffman-decoded (the pipeline's depth) */
static void job_read(const qs_cfg *g, qs_job *j, void (*host_wait)(void *arg), void *arg) {
	double t0 = now_ms();
	FILE *f; unsigned char *data; size_t len = 0;
	f = strcmp(j->in_name, "-") ? fopen(j->in_name, "rb") : stdin;
	if (!f) { fprintf(stderr, "%s: can't open input file \"%s\"\n", g->prog, j->in_name); j->rc = 1; return; }
	data = load_all(f, &len);
	if (f != stdin) fclose(f);
	if (!data) { fprintf(stderr, "%s: can't read input file \"%s\"\n", g->prog, j->in_name); j->rc = 1; return; }
#ifndef JPEGQS_NO_CUDA_RENDER
	if (!g->host_only) {
		jpegqs_cuda_file_info info; const char *why = "";
		int route = jpegqs_cuda_transcode_route(data, len, &why, &info);
		if (g->trace) fprintf(stderr, "jpegqs: %s: %s route (%s)\n", j->in_name, route == JPEGQS_ROUTE_DEVICE ? "device" : "host", why);
		if (route == JPEGQS_ROUTE_DEVICE) {
			j->data = data; j->len = len;
			if (g->verbose)
				fprintf(stderr, "%s: %ux%u, %d component(s), %s, restart interval %d\n", j->in_name, info.image_width,
						info.image_height, info.ncomp, info.progressive ? "progressive" : "sequential", info.restart_interval);
			j->t_read = now_ms() - t0;
			return;
		}
	} else if (g->trace) fprintf(stderr, "jpegqs: %s: host route (%s)\n", j->in_name, g->host_only);
#endif
	if (host_wait) host_wait(arg);
	job_decode(g, j, data, len, 1);
	j->t_read = now_ms() - t0;
}

/* the host route's middle stage: do_quantsmooth on the coefficients the reader decoded */
static void job_host_smooth(const qs_cfg *g, qs_job *j, double t0) {
	jpegqs_control_t opts = g->opts;
	if (do_quantsmooth(&j->im.cinfo, j->im.coef_arrays, &opts) < 0) j->rc = 2;
	j->t_smooth = now_ms() - t0;
}

#ifndef JPEGQS_NO_CUDA_RENDER
#define QS_BATCH_MAX 256                 /* device pairs per jpegqs_transcode_batch call */
/* the device route of m consecutive pairs in one call (jpegqs_transcode_batch); their -i lines are
 * printed pair by pair, and a pair that falls back takes the host route in its place, so stderr is
 * that of the pairs one after another */
static void job_smooth_device(const qs_cfg *g, qs_job *jobs, int m) {
	double t0 = now_ms(), t;
	const unsigned char *data[QS_BATCH_MAX]; size_t len[QS_BATCH_MAX]; unsigned char *out[QS_BATCH_MAX];
	size_t outlen[QS_BATCH_MAX]; int rc[QS_BATCH_MAX], k; const char *why[QS_BATCH_MAX]; char *log[QS_BATCH_MAX];
	jpegqs_control_t opts = g->opts;
	for (k = 0; k < m; k++) { data[k] = jobs[k].data; len[k] = jobs[k].len; }
	jpegqs_transcode_batch(m, data, len, g->copy, g->optimize, &opts, out, outlen, rc, why, log);
	t = now_ms() - t0;
	for (k = 0; k < m; k++) {
		qs_job *j = &jobs[k]; unsigned char *d = j->data;
		j->data = NULL;
		if (rc[k] != JPEGQS_TRANSCODE_FALLBACK) {
			if (log[k]) { fputs(log[k], stderr); free(log[k]); }
			free(d);
			j->out = out[k]; j->outlen = outlen[k];
			if (rc[k] < 0) j->rc = 2;
			j->t_smooth = t;
			continue;
		}
		/* damaged data (or a file the device route does not take after all): the host route gives
		 * the reader's recovery, warning count and messages */
		if (g->trace) fprintf(stderr, "jpegqs: %s: host route after all (%s)\n", j->in_name, why[k]);
		t0 = now_ms();
		job_decode(g, j, d, j->len, 0);
		if (!j->rc) job_host_smooth(g, j, t0);
	}
}
#endif

static void job_smooth(const qs_cfg *g, qs_job *j) {
#ifndef JPEGQS_NO_CUDA_RENDER
	if (j->data) { job_smooth_device(g, j, 1); return; }
#endif
	job_host_smooth(g, j, now_ms());
}

static void job_write(const qs_cfg *g, qs_job *j) {
	double t0 = now_ms();
	jq_image *im = &j->im;
	FILE *f; unsigned char *out = NULL; size_t outlen = 0; char err[256]; int io_err = 0, device = j->out != NULL;
#ifdef JPEGQS_NO_CUDA_RENDER
	if (g->ppm) { fprintf(stderr, "%s: --ppm needs the CUDA back end\n", g->prog); j->rc = 1; return; }
#else
	if (g->ppm) {                                       /* decode to RGB on the device */
		jpegqs_cuda_ctx *ctx = NULL; jpegqs_cuda_image ci; int c, nc = im->cinfo.num_components, rc;
		int16_t *bufs[MAX_COMPONENTS] = { 0 }; unsigned char *rgb; char hdr[64]; int hl;
		size_t npx = (size_t)im->cinfo.image_width * im->cinfo.image_height;
		if (jpegqs_cuda_create(g->cpu ? g->cpu - 1 : -1, &ctx)) {
			fprintf(stderr, "%s: CUDA back end unavailable: %s\n", g->prog, jpegqs_cuda_last_error(NULL));
			j->rc = 2; return;
		}
		memset(&ci, 0, sizeof(ci));
		ci.ncomp = nc; ci.is_ycbcr = im->cinfo.jpeg_color_space == JCS_YCbCr;
		ci.image_width = im->cinfo.image_width; ci.image_height = im->cinfo.image_height;
		for (c = 0; c < nc; c++) {
			jpeg_component_info *k = &im->cinfo.comp_info[c]; JDIMENSION y;
			size_t rowb = (size_t)k->width_in_blocks * sizeof(JBLOCK);
			bufs[c] = (int16_t*)malloc(rowb * k->height_in_blocks + 1);
			if (bufs[c]) for (y = 0; y < k->height_in_blocks; y++)
				memcpy((char*)bufs[c] + y * rowb, (*im->cinfo.mem->access_virt_barray)((j_common_ptr)&im->cinfo,
						im->coef_arrays[c], y, 1, FALSE)[0], rowb);
			ci.comp[c].coef = bufs[c]; ci.comp[c].wblk = k->width_in_blocks; ci.comp[c].hblk = k->height_in_blocks;
			ci.comp[c].h_samp = k->h_samp_factor; ci.comp[c].v_samp = k->v_samp_factor;
			ci.comp[c].has_qtbl = k->quant_table != NULL;
			if (k->quant_table) memcpy(ci.comp[c].quant, k->quant_table->quantval, sizeof(ci.comp[c].quant));
		}
		rgb = (unsigned char*)malloc(npx * 3 + 1);
		for (c = 0; c < nc; c++) if (!bufs[c]) rgb = (free(rgb), (unsigned char*)NULL);
		if (!rgb) {
			fprintf(stderr, "%s: out of memory\n", g->prog);
			for (c = 0; c < nc; c++) free(bufs[c]);
			jpegqs_cuda_destroy(ctx); j->rc = 1; return;
		}
		rc = jpegqs_cuda_render_rgb(ctx, &ci, 0, rgb, NULL);
		if (rc) fprintf(stderr, "%s: render failed (%d): %s\n", g->prog, rc, jpegqs_cuda_last_error(ctx));
		for (c = 0; c < nc; c++) free(bufs[c]);
		jpegqs_cuda_destroy(ctx);
		if (rc) { free(rgb); j->rc = 2; return; }
		if (nc == 1) { size_t k; for (k = 0; k < npx; k++) rgb[k] = rgb[3 * k]; }
		hl = snprintf(hdr, sizeof(hdr), "P%d\n%u %u\n255\n", nc == 1 ? 5 : 6, im->cinfo.image_width, im->cinfo.image_height);
		outlen = hl + npx * (nc == 1 ? 1 : 3);
		out = (unsigned char*)malloc(outlen);
		if (!out) { fprintf(stderr, "%s: out of memory\n", g->prog); free(rgb); j->rc = 1; return; }
		memcpy(out, hdr, hl); memcpy(out + hl, rgb, outlen - hl);
		free(rgb);
	} else
#endif
	if (device) { out = j->out; outlen = j->outlen; j->out = NULL; }     /* the device route wrote it */
	else if (jq_write(im, im->coef_arrays, g->optimize, &out, &outlen, err)) {
		fprintf(stderr, "%s: %s\n", g->prog, err); j->rc = 1; return;
	}
	/* the output is opened after the input was read, so it may name the same file */
	f = strcmp(j->out_name, "-") ? fopen(j->out_name, "wb") : stdout;
	if (!f) { fprintf(stderr, "%s: can't open output file \"%s\"\n", g->prog, j->out_name); free(out); j->rc = 1; return; }
	if (fwrite(out, 1, outlen, f) != outlen) io_err = 1;
	if (f != stdout ? fclose(f) != 0 : fflush(f) != 0) io_err = 1;      /* ENOSPC shows up at the flush */
	if (io_err) fprintf(stderr, "%s: error writing \"%s\"\n", g->prog, j->out_name);
	free(out);
	j->t_write = now_ms() - t0;
	if (g->verbose && device)
		fprintf(stderr, "wall time: read %.1f ms, device decode + do_quantsmooth + encode %.1f ms (includes waiting for "
				"CUDA start-up), write %.1f ms\n", j->t_read, j->t_smooth, j->t_write);
	else if (g->verbose) fprintf(stderr, "wall time: read + decode %.1f ms, do_quantsmooth %.1f ms (includes waiting for CUDA start-up), "
			"encode + write %.1f ms\n", j->t_read, j->t_smooth, j->t_write);
	/* the reference's exit status (quantsmooth.c:626): 2 when the codec met recoverable damage
	 * (libjpeg's num_warnings), else 0 - do_quantsmooth's "stopped early" value is not an error.
	 * A file with any warning never finishes on the device route. */
	j->rc = io_err ? 1 : !device && im->warnings ? 2 : 0;
}

static void job_release(qs_job *j) {
	if (j->have_im) { jq_free(&j->im); j->have_im = 0; }
	free(j->data); j->data = NULL;
	free(j->out); j->out = NULL;
}

/* one input -> one output, the stages in a row; returns the process exit status for this pair */
static int run_one(const qs_cfg *g, qs_job *j, int warm_ok) {
	int warm = 0;
#ifndef JPEGQS_NO_CUDA_RENDER
	pthread_t warm_th; int wflags = g->opts.flags;
	/* CUDA start-up (context + kernel image, a few hundred ms in a fresh process) overlaps with
	 * reading and Huffman-decoding the input */
	if (warm_ok && (g->opts.niter > 0 || (g->opts.flags & JPEGQS_UPSAMPLE_UV)) && !getenv("JPEGQS_NO_WARMUP"))
		warm = !pthread_create(&warm_th, NULL, warmup_thread, &wflags);
#endif
	(void)warm_ok;
	job_read(g, j, NULL, NULL);
	if (!j->rc) job_smooth(g, j);
#ifndef JPEGQS_NO_CUDA_RENDER
	if (warm) pthread_join(warm_th, NULL);
#endif
	(void)warm;
	if (!j->rc) job_write(g, j);
	job_release(j);
	return j->rc;
}

#ifndef JPEGQS_NO_CUDA_RENDER
/* --batch pipeline.  Reading and writing a file take longer than smoothing it, so several reader
 * threads (JPEGQS_BATCH_READERS, default 3) and writer threads (JPEGQS_BATCH_WRITERS, default 2)
 * work on different files at once while the calling thread keeps the device busy.  A reader does not
 * open an input that an earlier, unfinished pair is going to write.  How far readers run ahead:
 *   - a host-route pair is Huffman-decoded only once the pair `depth` places before it is written
 *     (an 8K image is 100 MB of coefficients);
 *   - a file is loaded once that pair is written, or while fewer than QS_AHEAD_PAIRS pairs before it
 *     are unwritten and the device-route pairs among them hold less than QS_AHEAD_BYTES of file
 *     bytes.  Device-route pairs hold only their bytes, so many of them can be read ahead, and the
 *     calling thread transcodes every read device-route pair that follows the next one in one call. */
#define QS_MAX_READERS 16
#define QS_AHEAD_PAIRS 128
#define QS_AHEAD_BYTES ((size_t)256 << 20)
typedef struct {
	const qs_cfg *g; qs_job *jobs; int n, next, wnext, depth, written;
	size_t held;                         /* file bytes of device-route pairs read and not yet written */
	pthread_mutex_t mu; pthread_cond_t cv;
} qs_pipe;

static void pipe_advance(qs_pipe *p, qs_job *j, int state) {
	pthread_mutex_lock(&p->mu);
	j->state = state;
	if (state == 3) { p->written++; p->held -= j->held; j->held = 0; }
	pthread_cond_broadcast(&p->cv); pthread_mutex_unlock(&p->mu);
}
static void pipe_wait(qs_pipe *p, qs_job *j, int state) {
	pthread_mutex_lock(&p->mu);
	while (j->state < state) pthread_cond_wait(&p->cv, &p->mu);
	pthread_mutex_unlock(&p->mu);
}
typedef struct { qs_pipe *p; qs_job *j; } qs_back;
static void wait_back(void *arg) { qs_back *b = (qs_back*)arg; pipe_wait(b->p, b->j, 3); }
static void *pipe_reader(void *arg) {
	qs_pipe *p = (qs_pipe*)arg; int i, k;
	for (;;) {
		pthread_mutex_lock(&p->mu); i = p->next++; pthread_mutex_unlock(&p->mu);
		if (i >= p->n) break;
		if (i >= p->depth) {
			qs_job *back = &p->jobs[i - p->depth];
			pthread_mutex_lock(&p->mu);
			while (back->state < 3 && (i - p->written >= QS_AHEAD_PAIRS || p->held >= QS_AHEAD_BYTES)) pthread_cond_wait(&p->cv, &p->mu);
			pthread_mutex_unlock(&p->mu);
		}
		for (k = 0; k < i; k++)
			if (strcmp(p->jobs[k].out_name, "-") && !strcmp(p->jobs[k].out_name, p->jobs[i].in_name)) pipe_wait(p, &p->jobs[k], 3);
		{
			qs_back back = { p, i >= p->depth ? &p->jobs[i - p->depth] : NULL };
			job_read(p->g, &p->jobs[i], back.j ? wait_back : NULL, &back);
		}
		pthread_mutex_lock(&p->mu);
		if (p->jobs[i].data) { p->jobs[i].held = p->jobs[i].len; p->held += p->jobs[i].len; }
		pthread_mutex_unlock(&p->mu);
		pipe_advance(p, &p->jobs[i], 1);
	}
	return NULL;
}
static void *pipe_writer(void *arg) {
	qs_pipe *p = (qs_pipe*)arg; int i, k;
	for (;;) {
		pthread_mutex_lock(&p->mu); i = p->wnext++; pthread_mutex_unlock(&p->mu);
		if (i >= p->n) break;
		pipe_wait(p, &p->jobs[i], 2);
		/* two pairs that name the same output are written in their order */
		for (k = 0; k < i; k++) if (!strcmp(p->jobs[k].out_name, p->jobs[i].out_name)) pipe_wait(p, &p->jobs[k], 3);
		if (!p->jobs[i].rc) job_write(p->g, &p->jobs[i]);
		job_release(&p->jobs[i]);
		pipe_advance(p, &p->jobs[i], 3);
	}
	return NULL;
}
/* returns the worst exit status of the pairs, -1 if no thread could be started (nothing done) */
static int run_pipeline(const qs_cfg *g, qs_job *jobs, int n) {
	qs_pipe p; pthread_t rd[QS_MAX_READERS], wr[QS_MAX_READERS]; int i, k, m, worst = 0, nrd = 3, nwr = 2, started = 0, writers = 0;
	const char *env = getenv("JPEGQS_BATCH_READERS");
	if (env && atoi(env) > 0) nrd = atoi(env);
	env = getenv("JPEGQS_BATCH_WRITERS");
	if (env && atoi(env) > 0) nwr = atoi(env);
	if (nrd > QS_MAX_READERS) nrd = QS_MAX_READERS;
	if (nwr > QS_MAX_READERS) nwr = QS_MAX_READERS;
	if (nrd > n) nrd = n;
	if (nwr > n) nwr = n;
	/* stdin is read and stdout written in the order of the pairs: one thread on that side then */
	for (i = 0; i < n; i++) { if (!strcmp(jobs[i].in_name, "-")) nrd = 1; if (!strcmp(jobs[i].out_name, "-")) nwr = 1; }
	p.g = g; p.jobs = jobs; p.n = n; p.next = 0; p.wnext = 0; p.depth = nrd + nwr + 1; p.written = 0; p.held = 0;
	pthread_mutex_init(&p.mu, NULL); pthread_cond_init(&p.cv, NULL);
	for (i = 0; i < nrd; i++) { if (pthread_create(&rd[started], NULL, pipe_reader, &p)) break; started++; }
	if (!started) { pthread_cond_destroy(&p.cv); pthread_mutex_destroy(&p.mu); return -1; }
	for (i = 0; i < nwr; i++) { if (pthread_create(&wr[writers], NULL, pipe_writer, &p)) break; writers++; }
	for (i = 0; i < n; i += m) {
		pipe_wait(&p, &jobs[i], 1);
		m = 1;
		if (!jobs[i].rc && jobs[i].data) {
			/* the device-route pairs right after this one that are already read go in the same call */
			pthread_mutex_lock(&p.mu);
			while (i + m < n && m < QS_BATCH_MAX && jobs[i + m].state >= 1 && !jobs[i + m].rc && jobs[i + m].data) m++;
			pthread_mutex_unlock(&p.mu);
			job_smooth_device(g, &jobs[i], m);
		} else if (!jobs[i].rc) job_smooth(g, &jobs[i]);
		for (k = i; k < i + m; k++) {
			if (writers) pipe_advance(&p, &jobs[k], 2);
			else {                                      /* no writer thread: write from here */
				if (!jobs[k].rc) job_write(g, &jobs[k]);
				job_release(&jobs[k]);
				pipe_advance(&p, &jobs[k], 3);
			}
		}
	}
	for (i = 0; i < started; i++) pthread_join(rd[i], NULL);
	for (i = 0; i < writers; i++) pthread_join(wr[i], NULL);
	pthread_cond_destroy(&p.cv); pthread_mutex_destroy(&p.mu);
	for (i = 0; i < n; i++) if (jobs[i].rc > worst) worst = jobs[i].rc;
	return worst;
}
#endif

int main(int argc, char **argv) {
	int optimize = 0, verbose = 0, info = 15, cpu = 0, copy = 2, quality = 3, niter = -1, cmd_flags = -1, threads = 0;
	int i, flags = 0, ppm = 0, batch = 0, status = 0;
	jpegqs_control_t opts;
	static const struct { char s; const char *l; int has_arg; } O[] = {
		{ 'o', "--optimize", 0 }, { 'v', "--verbose", 1 }, { 'i', "--info", 1 }, { 'n', "--niter", 1 },
		{ 'q', "--quality", 1 }, { 't', "--threads", 1 }, { 'f', "--flags", 1 }, { 'p', "--cpu", 1 }, { 'c', "--copy", 1 } };

	for (i = 1; i < argc; i++) {
		const char *a = argv[i], *val = NULL; int k, which = -1;
		if (a[0] != '-' || !a[1]) break;
		if (!strcmp(a, "--")) { i++; break; }
		if (!strcmp(a, "--ppm")) { ppm = 1; continue; }
		if (!strcmp(a, "--batch")) { batch = 1; continue; }
		for (k = 0; k < (int)(sizeof(O) / sizeof(O[0])); k++) {
			if (a[1] != '-' && a[1] == O[k].s) { which = k; if (a[2]) val = a + 2; break; }
			if (!strcmp(a, O[k].l)) { which = k; break; }
		}
		if (which < 0) return usage(argv[0]);
		if (O[which].has_arg) {
			if (!val) { if (++i >= argc) return usage(argv[0]); val = argv[i]; }
			if ((unsigned)(val[0] - '0') > 9) return usage(argv[0]);
		} else if (val) return usage(argv[0]);
		switch (O[which].s) {
			case 'o': optimize = 1; break;
			case 'v': verbose = atoi(val); break;
			case 'i': info = atoi(val); break;
			case 'n': niter = atoi(val); break;
			case 'q': quality = atoi(val); break;
			case 't': threads = atoi(val); break;
			case 'f': cmd_flags = atoi(val) & JPEGQS_FLAGS_MASK; break;
			case 'p': cpu = atoi(val); if (cpu > JPEGQS_CPU_MASK) cpu = JPEGQS_CPU_MASK; break;
			case 'c': copy = atoi(val); break;
		}
	}
	if (batch ? (argc - i < 2 || ((argc - i) & 1)) : argc - i != 2) return usage(argv[0]);

	if (quality < 3) { flags |= JPEGQS_LOW_QUALITY; quality += 4; }      /* quantsmooth.c:380-393 */
	if (quality >= 4) flags |= JPEGQS_DIAGONALS;
	if (quality >= 5) flags |= JPEGQS_JOINT_YUV;
	if (quality >= 6) flags |= JPEGQS_UPSAMPLE_UV;
	memset(&opts, 0, sizeof(opts));
	opts.niter = niter >= 0 ? niter : 3;
	opts.flags = (cmd_flags >= 0 ? cmd_flags : flags) | JPEGQS_TRANSCODE;
	opts.flags |= cpu << JPEGQS_CPU_SHIFT;
	opts.flags |= info << JPEGQS_INFO_SHIFT;
	opts.threads = threads;
	if (threads > 0) jq_set_threads(threads);

	/* --batch: any number of "input output" pairs in one process, so that CUDA start-up (context and
	 * kernel image, seconds in a fresh process) is paid once; the exit status is the worst of the pairs */
	{
		qs_cfg g; qs_job *jobs; int n = (argc - i) / 2, k;
		const char *gpus = getenv("JPEGQS_GPUS");
		g.prog = argv[0]; g.opts = opts; g.copy = copy; g.optimize = optimize; g.verbose = verbose; g.ppm = ppm; g.cpu = cpu;
		g.trace = getenv("JPEGQS_CODEC_TRACE") != NULL;
		/* the device route where the pair reaches the device anyway (the warm-up's condition) and
		 * its output is a JPEG file; JPEGQS_HOST_CODEC=1 keeps every pair on the host codec */
		g.host_only = ppm ? "--ppm" : !(opts.niter > 0 || (opts.flags & JPEGQS_UPSAMPLE_UV)) ? "nothing to smooth" :
				gpus && *gpus ? "JPEGQS_GPUS" : getenv("JPEGQS_HOST_CODEC") ? "JPEGQS_HOST_CODEC" : NULL;
		jobs = (qs_job*)calloc((size_t)n, sizeof(qs_job));
		if (!jobs) { fprintf(stderr, "%s: out of memory\n", argv[0]); return 1; }
		for (k = 0; k < n; k++) { jobs[k].in_name = argv[i + 2 * k]; jobs[k].out_name = argv[i + 2 * k + 1]; }
		k = 0;
#ifdef __GLIBC__
		/* the 100 MB coefficient arrays of one pair become those of the next: kept in the heap
		 * they are cleared by a memset instead of being unmapped and page-faulted in again
		 * (one arena: the reader thread's allocations must come from that heap too) */
		if (n > 1) { mallopt(M_MMAP_THRESHOLD, 1 << 30); mallopt(M_TRIM_THRESHOLD, 1 << 30); mallopt(M_ARENA_MAX, 1); }
#endif
#ifndef JPEGQS_NO_CUDA_RENDER
		/* (--ppm renders on the device inside the write stage: those pairs stay in a row) */
		if (n > 1 && !ppm && !getenv("JPEGQS_NO_PIPELINE")) {
			int rc;
			/* the first pair alone, with the CUDA warm-up beside its decode; the rest as a pipeline */
			double t0;
			status = run_one(&g, &jobs[0], 1);
			t0 = now_ms();
			rc = run_pipeline(&g, jobs + 1, n - 1);
			if (rc > status) status = rc;
			k = rc < 0 ? 1 : n;
			if (verbose && rc >= 0) fprintf(stderr, "batch: %d pairs after the first in %.1f ms (pipeline)\n", n - 1, now_ms() - t0);
		}
#endif
		if (k < n) {
			double t0 = 0; int first = k;
			for (; k < n; k++) {
				int rc = run_one(&g, &jobs[k], status == 0); if (rc > status) status = rc;
				if (k == 0) t0 = now_ms();
			}
			if (verbose && n > 1 && first == 0) fprintf(stderr, "batch: %d pairs after the first in %.1f ms (one after the other)\n", n - 1, now_ms() - t0);
		}
		free(jobs);
	}
	return status;
}
