/*
 * do_quantsmooth.c - the libjpeg-facing entry points of libjpegqs (include/libjpegqs.h),
 * kept in C like the reference's host code.  They do what the reference driver does on
 * the libjpeg side of the boundary (reference quantsmooth.h:2404-2453 argument handling,
 * 2836-2876 result plumbing, 2880-2904 decode helpers) and hand the arithmetic to the CUDA
 * back end through the C ABI of include/jpegqs_cuda.h: the block rows of libjpeg's virtual
 * arrays (access_virt_barray, one row contiguous, rows not necessarily adjacent - SURVEY.md 8b)
 * are passed as row-pointer tables; the back end gathers them into its pinned staging memory
 * band by band on worker threads while the first bands are already being smoothed, and
 * scatters the results back the same way (jpegqs_cuda_comp.rows).
 *
 * There is no CPU implementation here: if the CUDA back end cannot run, the call reports
 * the error on stderr and returns a negative code with the coefficients untouched.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <jpeglib.h>
#include "libjpegqs.h"
#include "jpegqs_cuda.h"
#include "jpegcoef.h"

#ifndef JPEGQS_NO_LOG
#define WITH_LOG
#include <sys/time.h>
static int64_t now_usec(void) {
	struct timeval tv; gettimeofday(&tv, NULL);
	return tv.tv_sec * (int64_t)1000000 + tv.tv_usec;
}
#endif

#if !defined(TRANSCODE_ONLY) && !defined(JPEG_INTERNALS)
/* What the decode helpers need from libjpeg beyond jpeglib.h (the reference declares the same
 * things by hand, quantsmooth.h:33-61): two decoder states, the four module initialisers that
 * re-arm the output side after the coefficient arrays were replaced (2861-2876), and - for
 * libjpeg-turbo, whose IDCT stops at master->last_MCU_col - the private master record. */
#define DSTATE_SCANNING 205
#define DSTATE_RAW_OK 206
#define QS_WEAK __attribute__((weak))
EXTERN(void) jinit_d_main_controller(j_decompress_ptr, boolean) QS_WEAK;
EXTERN(void) jinit_inverse_dct(j_decompress_ptr) QS_WEAK;
EXTERN(void) jinit_upsampler(j_decompress_ptr) QS_WEAK;
EXTERN(void) jinit_color_deconverter(j_decompress_ptr) QS_WEAK;
struct jpeg_decomp_master {
	void (*prepare_for_output_pass)(j_decompress_ptr);
	void (*finish_output_pass)(j_decompress_ptr);
	boolean is_dummy_pass;
#ifdef LIBJPEG_TURBO_VERSION
#if LIBJPEG_TURBO_VERSION_NUMBER >= 2001090
	boolean lossless;
#endif
	JDIMENSION first_iMCU_col, last_iMCU_col;
	JDIMENSION first_MCU_col[MAX_COMPONENTS];
	JDIMENSION last_MCU_col[MAX_COMPONENTS];
	boolean jinit_upsampler_no_alloc;
#if LIBJPEG_TURBO_VERSION_NUMBER >= 2000090
	JDIMENSION last_good_iMCU_row;
#endif
#endif
};
#endif
#ifndef TRANSCODE_ONLY
/* The library does not pull in a libjpeg of its own: the application that calls the decode
 * helpers has one loaded, and these weak references bind to it.  A process without libjpeg
 * (the Python tests, a transcoder built on another codec) can still load the library; the
 * helpers then report the missing symbols instead of crashing. */
#ifndef QS_WEAK
#define QS_WEAK __attribute__((weak))
#endif
EXTERN(boolean) jpeg_start_decompress(j_decompress_ptr) QS_WEAK;
EXTERN(boolean) jpeg_input_complete(j_decompress_ptr) QS_WEAK;
EXTERN(boolean) jpeg_start_output(j_decompress_ptr, int) QS_WEAK;
EXTERN(boolean) jpeg_finish_output(j_decompress_ptr) QS_WEAK;
EXTERN(jvirt_barray_ptr *) jpeg_read_coefficients(j_decompress_ptr) QS_WEAK;
EXTERN(boolean) jpeg_finish_decompress(j_decompress_ptr) QS_WEAK;
#endif

/* one lazily created context per device ordinal.  The reference function is re-entrant; this one
 * shares a device context (arena, staging, streams) between callers, so calls are serialised
 * by a lock - like the reference's own plugin does around it (irfanview/plugin.c:148-162). */
#include <pthread.h>
#define QS_MAX_DEVICES 16
static jpegqs_cuda_ctx *g_ctx[QS_MAX_DEVICES + 1];
static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;

/* JPEGQS_GPUS=n (or "all"): images large enough are sharded by MCU rows over n devices of this
 * process (include/jpegqs_cuda.h jpegqs_cuda_run_host_multi; SURVEY.md 8e).  The reference's
 * knob for parallelism is opts->threads (quantsmooth.h:2467-2472), which callers set to CPU
 * counts - an environment variable cannot be misread that way.  Not with a progress callback
 * (its sequence is per component, quantsmooth.h:2656-2664) and not with an explicit device. */
static jpegqs_cuda_multi *g_multi;
static int g_multi_tried;
static jpegqs_cuda_multi *get_multi(void) {
	if (!g_multi_tried) {
		const char *e = getenv("JPEGQS_GPUS");
		g_multi_tried = 1;
		if (e && *e) {
			int n = !strcmp(e, "all") ? 0 : atoi(e);
			if ((n > 1 || !strcmp(e, "all")) && jpegqs_cuda_multi_create(n, NULL, &g_multi)) {
				fprintf(stderr, "jpegqs: JPEGQS_GPUS=%s ignored: %s\n", e, jpegqs_cuda_last_error(NULL));
				g_multi = NULL;
			}
		}
	}
	return g_multi;
}

static jpegqs_cuda_ctx *get_ctx_quiet(int ordinal_plus1) {
	int slot = ordinal_plus1 < 0 || ordinal_plus1 > QS_MAX_DEVICES ? 0 : ordinal_plus1;
	if (!g_ctx[slot] && jpegqs_cuda_create(slot ? slot - 1 : -1, &g_ctx[slot])) g_ctx[slot] = NULL;
	return g_ctx[slot];
}
static void report_unavailable(void) {
	fprintf(stderr, "jpegqs: CUDA back end unavailable: %s\n", jpegqs_cuda_last_error(NULL));
}
static jpegqs_cuda_ctx *get_ctx(int ordinal_plus1) {
	jpegqs_cuda_ctx *ctx = get_ctx_quiet(ordinal_plus1);
	if (!ctx) report_unavailable();
	return ctx;
}

/* Extension (include/libjpegqs.h): create the context do_quantsmooth(flags) will use.  CUDA
 * initialisation + loading the kernels take a few hundred ms in a fresh process - as long as
 * decoding a large file - so a tool can run this on a second thread while it parses its input
 * (csrc/jpegqs.c does).  Silent on failure: the real call reports. */
JPEGQS_ATTR
int jpegqs_warmup(int flags) {
	int slot = (flags >> JPEGQS_CPU_SHIFT) & JPEGQS_CPU_MASK, ok;
	pthread_mutex_lock(&g_lock);
	if (!g_ctx[slot] && jpegqs_cuda_create(slot ? slot - 1 : -1, &g_ctx[slot])) g_ctx[slot] = NULL;
	ok = g_ctx[slot] != NULL;
	pthread_mutex_unlock(&g_lock);
	return ok ? 0 : JPEGQS_ERR_CUDA;
}


#ifdef WITH_LOG
/* The -i lines (JPEGQS_INFO_*), the same for do_quantsmooth and jpegqs_transcode.  Before anything is
 * touched: component tables and sampling, the quantization tables. */
static void log_head(FILE *f, j_decompress_ptr srcinfo, int flags) {
	jpeg_component_info *comp = srcinfo->comp_info; int ci, i, k;
	if (flags & JPEGQS_INFO_COMP1)
		for (ci = 0; ci < srcinfo->num_components; ci++)
			fprintf(f, "component[%i] : table %i, samp %ix%i\n", ci, comp[ci].quant_tbl_no,
					comp[ci].h_samp_factor, comp[ci].v_samp_factor);
	if (flags & JPEGQS_INFO_QUANT)
		for (i = 0; i < NUM_QUANT_TBLS; i++) {
			JQUANT_TBL *t = srcinfo->quant_tbl_ptrs[i];
			if (!t) continue;
			fprintf(f, "quant[%i]:\n", i);
			for (k = 0; k < DCTSIZE2; k++) {
				fprintf(f, "%04x ", t->quantval[k]);
				if ((k & 7) == 7) fprintf(f, "\n");
			}
		}
}
/* once the device is reached: the back end, the component sizes (quantsmooth.h:2569-2572) */
static void log_device(FILE *f, j_decompress_ptr srcinfo, int flags, jpegqs_cuda_ctx *ctx, jpegqs_cuda_multi *multi) {
	jpeg_component_info *comp = srcinfo->comp_info; int ci;
	if (flags & JPEGQS_INFO_CPU) {
		if (multi) fprintf(f, "SIMD type: CUDA sm_90a (%s x %d)\n", jpegqs_cuda_device_name(ctx), jpegqs_cuda_multi_devices(multi));
		else fprintf(f, "SIMD type: CUDA sm_90a (%s)\n", jpegqs_cuda_device_name(ctx));
	}
	if (flags & JPEGQS_INFO_COMP2)
		for (ci = 0; ci < srcinfo->num_components; ci++) if (comp[ci].quant_table)
			fprintf(f, "component[%i] : size %ix%i\n", ci, comp[ci].width_in_blocks, comp[ci].height_in_blocks);
}
/* at the end of a run that did not stop */
static void log_time(FILE *f, int flags, int64_t usec, jpegqs_cuda_ctx *ctx) {
	if (flags & JPEGQS_INFO_TIME) {
		fprintf(f, "quantsmooth: %.3fms\n", usec * 0.001);
		fprintf(f, "quantsmooth (device kernels): %.3fms\n", jpegqs_cuda_last_device_ms(ctx));
	}
}
#endif

/* YCbCr with 1x1 chroma under JOINT_YUV / UPSAMPLE_UV: the chroma feed from a down-sampled luma */
static int needs_downsample(j_decompress_ptr srcinfo, int flags) {
	jpeg_component_info *comp = srcinfo->comp_info;
	return flags & (JPEGQS_JOINT_YUV | JPEGQS_UPSAMPLE_UV) && srcinfo->jpeg_color_space == JCS_YCbCr &&
			srcinfo->num_components >= 3 && comp[1].h_samp_factor == 1 && comp[1].v_samp_factor == 1 &&
			comp[2].h_samp_factor == 1 && comp[2].v_samp_factor == 1;
}
/* 0: do_quantsmooth returns at once and touches nothing (quantsmooth.h:2447-2458) */
static int smooths(j_decompress_ptr srcinfo, int flags, int niter) {
	if (srcinfo->num_components < 1 || srcinfo->num_components > JPEGQS_CUDA_MAX_COMP) return 0;
	if (niter > JPEGQS_ITER_MAX) niter = JPEGQS_ITER_MAX;
	return niter > 0 || (flags & JPEGQS_UPSAMPLE_UV && needs_downsample(srcinfo, flags));
}

/* Extension (include/libjpegqs.h): the jpegqs tool's device route, n files in shared launches
 * (jpegqs_cuda_transcode_batch).  The same context, lock, device selection and messages as
 * do_quantsmooth, and for each file the same -i lines in the same order as a call for that file
 * alone, files in their order.  The time line of a file gives the wall time of the whole call and the
 * device-kernel line the run_async time of its last sub-batch (jpegqs_cuda_last_device_ms): with the
 * default device budget one call is one sub-batch unless its files need more than half the device's
 * free memory.  A file that falls back prints nothing.  The coefficients never leave the device. */
JPEGQS_ATTR
int jpegqs_transcode_batch(int n, const unsigned char *const *data, const size_t *len, int copy, int optimize,
		jpegqs_control_t *opts, unsigned char **out, size_t *outlen, int *rc, const char **reason, char **log) {
	jq_image im; char err[256]; int flags = opts->flags, i, m = 0, ret = 0; jpegqs_cuda_ctx *ctx;
	int *smooth, *idx, *brc; FILE **f; char **buf; size_t *blen; const unsigned char **bdata; size_t *blens;
	jpegqs_cuda_transcode_result *res;
#ifdef WITH_LOG
	int64_t t0 = 0, usec = 0;
#endif
	if (n <= 0) return 0;
	smooth = (int*)calloc((size_t)n, sizeof(int)); idx = (int*)calloc((size_t)n, sizeof(int)); brc = (int*)calloc((size_t)n, sizeof(int));
	f = (FILE**)calloc((size_t)n, sizeof(FILE*)); buf = (char**)calloc((size_t)n, sizeof(char*)); blen = (size_t*)calloc((size_t)n, sizeof(size_t));
	bdata = (const unsigned char**)calloc((size_t)n, sizeof(*bdata)); blens = (size_t*)calloc((size_t)n, sizeof(size_t));
	res = (jpegqs_cuda_transcode_result*)calloc((size_t)n, sizeof(*res));
	if (!smooth || !idx || !brc || !f || !buf || !blen || !bdata || !blens || !res) {
		for (i = 0; i < n; i++) { out[i] = NULL; outlen[i] = 0; rc[i] = JPEGQS_TRANSCODE_FALLBACK; reason[i] = "out of memory"; if (log) log[i] = NULL; }
		ret = JPEGQS_TRANSCODE_FALLBACK; goto done;
	}
	for (i = 0; i < n; i++) {
		out[i] = NULL; outlen[i] = 0; reason[i] = ""; rc[i] = JPEGQS_TRANSCODE_OK; if (log) log[i] = NULL;
		/* what do_quantsmooth would be handed: the frame, quant tables and colour space of the file */
		if (jq_read_markers(data[i], len[i], 0, &im, err)) { reason[i] = "the reader rejects the file"; rc[i] = JPEGQS_TRANSCODE_FALLBACK; continue; }
		smooth[i] = smooths(&im.cinfo, flags, opts->niter);
		f[i] = open_memstream(&buf[i], &blen[i]);
		if (!f[i]) { jq_free(&im); reason[i] = "out of memory"; rc[i] = JPEGQS_TRANSCODE_FALLBACK; continue; }
#ifdef WITH_LOG
		log_head(f[i], &im.cinfo, flags);
#endif
		idx[m] = i; bdata[m] = data[i]; blens[m] = len[i]; m++;
		jq_free(&im);
	}
	pthread_mutex_lock(&g_lock);
	ctx = get_ctx_quiet((flags >> JPEGQS_CPU_SHIFT) & JPEGQS_CPU_MASK);
	if (!ctx) {
		for (i = 0; i < m; i++) {
			int k = idx[i];
			/* do_quantsmooth would not reach the device: the host route gives the file without one */
			if (!smooth[k]) { rc[k] = JPEGQS_TRANSCODE_FALLBACK; reason[k] = "no CUDA device, and nothing to smooth"; continue; }
			rc[k] = JPEGQS_ERR_CUDA;
			fprintf(f[k], "jpegqs: CUDA back end unavailable: %s\n", jpegqs_cuda_last_error(NULL));
		}
	} else if (m) {
		int r;
#ifdef WITH_LOG
		for (i = 0; i < m; i++) {
			if (!smooth[idx[i]]) continue;
			if (jq_read_markers(data[idx[i]], len[idx[i]], 0, &im, err)) continue;
			log_device(f[idx[i]], &im.cinfo, flags, ctx, NULL);
			jq_free(&im);
		}
		t0 = now_usec();
#endif
		r = jpegqs_cuda_transcode_batch(ctx, m, bdata, blens, flags, opts->niter, optimize, copy, 0, brc, res);
#ifdef WITH_LOG
		usec = now_usec() - t0;
#endif
		for (i = 0; i < m; i++) {
			int k = idx[i];
			rc[k] = r < 0 ? r : brc[i];
			if (rc[k] == JPEGQS_TRANSCODE_FALLBACK) { reason[k] = res[i].reason; continue; }
			if (rc[k] < 0) { fprintf(f[k], "jpegqs: CUDA back end failed (%d): %s\n", rc[k], jpegqs_cuda_last_error(ctx)); continue; }
#ifdef WITH_LOG
			if (smooth[k] && !res[i].stop) log_time(f[k], flags, usec, ctx);
#endif
			out[k] = res[i].data; outlen[k] = res[i].len;
		}
	}
	for (i = 0; i < m; i++) {
		int k = idx[i];
		fclose(f[k]); f[k] = NULL;
		if (rc[k] == JPEGQS_TRANSCODE_FALLBACK || !blen[k]) { free(buf[k]); buf[k] = NULL; }
		if (!log) { if (buf[k]) fwrite(buf[k], 1, blen[k], stderr); free(buf[k]); }
		else log[k] = buf[k];
		buf[k] = NULL;
	}
	pthread_mutex_unlock(&g_lock);
done:
	free(smooth); free(idx); free(brc); free(f); free(buf); free(blen); free(bdata); free(blens); free(res);
	return ret;
}

/* Extension (include/libjpegqs.h): one file, the batch of one. */
JPEGQS_ATTR
int jpegqs_transcode(const unsigned char *data, size_t len, int copy, int optimize, jpegqs_control_t *opts,
		unsigned char **out, size_t *outlen, const char **reason) {
	int rc = 0;
	jpegqs_transcode_batch(1, &data, &len, copy, optimize, opts, out, outlen, &rc, reason, NULL);
	return rc;
}

/* Block-row table of one virtual array: libjpeg keeps a whole-image coefficient array in memory
 * as separately allocated row groups (jmemmgr.c alloc_barray), and access_virt_barray returns
 * pointers into them.  The reference calls it once per row from inside its OpenMP loops
 * (quantsmooth.h:2592-2594, 2706-2710); here every row is touched once, in order, on the
 * calling thread and the pointers are handed to the back end, whose worker threads gather /
 * scatter the rows while the device is already working.  A memory manager that pages the array
 * through a backing store would hand out the same buffer for different rows: then (distinct ==
 * 0) the rows are copied one by one on this thread instead. */
static int16_t **row_table(j_decompress_ptr cinfo, jvirt_barray_ptr arr, JDIMENSION h, int *distinct) {
	JDIMENSION y; int16_t **t = (int16_t**)malloc(sizeof(int16_t*) * (h ? h : 1));
	if (!t) return NULL;
	for (y = 0; y < h; y++)
		t[y] = (int16_t*)(*cinfo->mem->access_virt_barray)((j_common_ptr)cinfo, arr, y, 1, TRUE)[0];
	*distinct = 1;
	if (h > 1) {
		/* all pointers distinct <=> the array is fully resident (rows of a backing-store window repeat) */
		int16_t **u = (int16_t**)malloc(sizeof(int16_t*) * h);
		if (!u) { free(t); return NULL; }
		memcpy(u, t, sizeof(int16_t*) * h);
		{	/* shell sort: no libc comparator call per element, h <= 65500/8 */
			JDIMENSION gap, i, j;
			for (gap = h / 2; gap; gap /= 2)
				for (i = gap; i < h; i++) {
					int16_t *v = u[i];
					for (j = i; j >= gap && (uintptr_t)u[j - gap] > (uintptr_t)v; j -= gap) u[j] = u[j - gap];
					u[j] = v;
				}
		}
		for (y = 1; y < h; y++) if (u[y] == u[y - 1]) { *distinct = 0; break; }
		free(u);
	}
	return t;
}

JPEGQS_ATTR
int do_quantsmooth(j_decompress_ptr srcinfo, jvirt_barray_ptr *coef_arrays, jpegqs_control_t *opts) {
	jpegqs_cuda_image img; jpegqs_cuda_ctx *ctx; jpegqs_cuda_multi *multi = NULL;
	jpeg_component_info *comp = srcinfo->comp_info;
	int ci, i, ret, ncomp = srcinfo->num_components;
	int need_downsample, flags = opts->flags, resident = 1, will_upsample;
	int16_t **rows[JPEGQS_CUDA_MAX_COMP], **rows_up[2] = { NULL, NULL };
	int16_t *flat[JPEGQS_CUDA_MAX_COMP], *flat_up[2] = { NULL, NULL };
	jvirt_barray_ptr up[2] = { NULL, NULL };
	JDIMENSION y;
#ifdef WITH_LOG
	int64_t t0 = 0;
	log_head(stderr, srcinfo, flags);
	if (flags & JPEGQS_INFO_TIME) t0 = now_usec();
#endif
	if (ncomp < 1 || ncomp > JPEGQS_CUDA_MAX_COMP) return 0;

	/* same early exit as the reference (quantsmooth.h:2447-2458): nothing is touched */
	need_downsample = needs_downsample(srcinfo, flags);
	if (!smooths(srcinfo, flags, opts->niter)) return 0;
	will_upsample = need_downsample && flags & JPEGQS_UPSAMPLE_UV &&
			(comp[0].h_samp_factor != 1 || comp[0].v_samp_factor != 1);

	pthread_mutex_lock(&g_lock);
	if (!opts->progress && !((flags >> JPEGQS_CPU_SHIFT) & JPEGQS_CPU_MASK)) multi = get_multi();
	ctx = multi ? jpegqs_cuda_multi_ctx(multi, 0) : get_ctx((flags >> JPEGQS_CPU_SHIFT) & JPEGQS_CPU_MASK);
	if (!ctx) { pthread_mutex_unlock(&g_lock); return JPEGQS_ERR_CUDA; }
#ifdef WITH_LOG
	log_device(stderr, srcinfo, flags, ctx, multi);
#endif

	memset(&img, 0, sizeof(img));
	memset(rows, 0, sizeof(rows)); memset(flat, 0, sizeof(flat));
	img.ncomp = ncomp;
	img.is_ycbcr = srcinfo->jpeg_color_space == JCS_YCbCr;
	img.image_width = srcinfo->image_width; img.image_height = srcinfo->image_height;
	ret = JPEGQS_ERR_CUDA;
	if (will_upsample) {
		/* the luma-sized chroma arrays of quantsmooth.h:2700-2702: requested up front so that
		 * their rows exist while the device results stream back (if the run stops they stay
		 * unused in the image pool, which libjpeg frees with the image) */
		JDIMENSION W0 = comp[0].width_in_blocks, H0 = comp[0].height_in_blocks;
		for (i = 0; i < 2; i++)
			up[i] = (*srcinfo->mem->request_virt_barray)((j_common_ptr)srcinfo, JPOOL_IMAGE, FALSE, W0, H0, 1);
		(*srcinfo->mem->realize_virt_arrays)((j_common_ptr)srcinfo);
		if (!up[0] || !up[1]) goto done;               /* a memory manager that returns instead of error_exit */
	}
	for (ci = 0; ci < ncomp; ci++) {
		jpegqs_cuda_comp *c = &img.comp[ci]; int distinct = 1;
		c->wblk = comp[ci].width_in_blocks; c->hblk = comp[ci].height_in_blocks;
		c->h_samp = comp[ci].h_samp_factor; c->v_samp = comp[ci].v_samp_factor;
		c->has_qtbl = comp[ci].quant_table != NULL;
		if (c->has_qtbl) memcpy(c->quant, comp[ci].quant_table->quantval, sizeof(c->quant));
		rows[ci] = row_table(srcinfo, coef_arrays[ci], c->hblk, &distinct);
		if (!rows[ci]) goto done;
		resident &= distinct;
	}
	if (will_upsample) for (i = 0; i < 2; i++) {
		int distinct = 1;
		rows_up[i] = row_table(srcinfo, up[i], comp[0].height_in_blocks, &distinct);
		if (!rows_up[i]) goto done;
		resident &= distinct;
	}
	if (resident) {
		for (ci = 0; ci < ncomp; ci++) img.comp[ci].rows = rows[ci];
		for (i = 0; i < 2; i++) img.comp[1 + i].rows_up = rows_up[i];
	} else {
		/* paged arrays: one row at a time on this thread, into flat buffers the back end stages */
		for (ci = 0; ci < ncomp; ci++) {
			jpegqs_cuda_comp *c = &img.comp[ci]; size_t rowb = (size_t)c->wblk * sizeof(JBLOCK);
			flat[ci] = (int16_t*)malloc(rowb * c->hblk + 1);
			if (!flat[ci]) goto done;
			c->coef = flat[ci];
			for (y = 0; y < c->hblk; y++) {
				JBLOCKARRAY r = (*srcinfo->mem->access_virt_barray)((j_common_ptr)srcinfo, coef_arrays[ci], y, 1, TRUE);
				memcpy((char*)flat[ci] + y * rowb, r[0], rowb);
			}
		}
		if (will_upsample) for (i = 0; i < 2; i++) {
			flat_up[i] = (int16_t*)malloc((size_t)img.comp[0].wblk * img.comp[0].hblk * sizeof(JBLOCK) + 1);
			if (!flat_up[i]) goto done;
			img.comp[1 + i].coef_up = flat_up[i];
		}
	}

	if (multi) ret = jpegqs_cuda_run_host_multi(multi, &img, flags & JPEGQS_FLAGS_MASK, opts->niter);
	else ret = jpegqs_cuda_run_host(ctx, &img, flags & JPEGQS_FLAGS_MASK, opts->niter, opts->progprec,
			opts->progress, opts->userdata);
	if (ret < 0) {
		fprintf(stderr, "jpegqs: CUDA back end failed (%d): %s\n", ret,
				multi ? jpegqs_cuda_multi_last_error(multi) : jpegqs_cuda_last_error(ctx));
		goto done;
	}

	if (!resident) {
		for (ci = 0; ci < ncomp; ci++) {
			jpegqs_cuda_comp *c = &img.comp[ci]; size_t rowb = (size_t)c->wblk * sizeof(JBLOCK);
			if (img.upsampled && (ci == 1 || ci == 2)) continue;
			for (y = 0; y < c->hblk; y++) {
				JBLOCKARRAY r = (*srcinfo->mem->access_virt_barray)((j_common_ptr)srcinfo, coef_arrays[ci], y, 1, TRUE);
				memcpy(r[0], (char*)flat[ci] + y * rowb, rowb);
			}
		}
		if (img.upsampled) for (i = 0; i < 2; i++) {
			size_t rowb = (size_t)comp[0].width_in_blocks * sizeof(JBLOCK);
			for (y = 0; y < comp[0].height_in_blocks; y++) {
				JBLOCKARRAY r = (*srcinfo->mem->access_virt_barray)((j_common_ptr)srcinfo, up[i], y, 1, TRUE);
				memcpy(r[0], (char*)flat_up[i] + y * rowb, rowb);
			}
		}
	}
	if (img.upsampled) {                               /* quantsmooth.h:2836-2849 */
		JDIMENSION W0 = comp[0].width_in_blocks, H0 = comp[0].height_in_blocks;
		for (i = 0; i < 2; i++) {
			coef_arrays[1 + i] = up[i];
			comp[1 + i].width_in_blocks = W0; comp[1 + i].height_in_blocks = H0;
		}
		srcinfo->max_h_samp_factor = 1; srcinfo->max_v_samp_factor = 1;
		comp[0].h_samp_factor = 1; comp[0].v_samp_factor = 1;
	}
	for (i = 0; i < NUM_QUANT_TBLS; i++) {             /* quantsmooth.h:2851-2859 */
		JQUANT_TBL *t = srcinfo->quant_tbl_ptrs[i]; int k;
		if (t) for (k = 0; k < DCTSIZE2; k++) t->quantval[k] = 1;
	}
	for (ci = 0; ci < ncomp; ci++) {
		JQUANT_TBL *t = comp[ci].quant_table; int k;
		if (t) for (k = 0; k < DCTSIZE2; k++) t->quantval[k] = 1;
	}
#ifndef TRANSCODE_ONLY
	if (!(flags & JPEGQS_TRANSCODE)) {                 /* quantsmooth.h:2861-2876 */
		if (!jinit_inverse_dct || !jinit_upsampler || !jinit_color_deconverter || !jinit_d_main_controller) {
			fprintf(stderr, "jpegqs: no libjpeg in this process to re-arm the decoder (JPEGQS_TRANSCODE not set)\n");
			ret = JPEGQS_ERR_ARG;
		} else {
		if (img.upsampled) {
#ifdef LIBJPEG_TURBO_VERSION
			srcinfo->master->last_MCU_col[1] = srcinfo->master->last_MCU_col[0];
			srcinfo->master->last_MCU_col[2] = srcinfo->master->last_MCU_col[0];
#endif
			jinit_color_deconverter(srcinfo);
			jinit_upsampler(srcinfo);
			jinit_d_main_controller(srcinfo, FALSE);
			srcinfo->input_iMCU_row = (srcinfo->output_height + DCTSIZE - 1) / DCTSIZE;
		}
		jinit_inverse_dct(srcinfo);
		}
	}
#endif
#ifdef WITH_LOG
	if (!ret) log_time(stderr, flags, now_usec() - t0, ctx);
#endif
done:
	for (ci = 0; ci < ncomp; ci++) { free(rows[ci]); free(flat[ci]); }
	for (i = 0; i < 2; i++) { free(rows_up[i]); free(flat_up[i]); }
	pthread_mutex_unlock(&g_lock);
	return ret;
}

/* The reference's SIMD_SELECT build (Makefile:176-185) links one do_quantsmooth per
 * instruction-set tier and picks one at run time (libjpegqs.c:80-156, declarations 38-58).  The
 * CUDA back end occupies exactly that slot: with these four names a caller compiled as
 * `quantsmooth.c -DSIMD_SELECT` (which includes the dispatcher libjpegqs.c) links against this
 * library unchanged, whichever tier its cpuid logic picks.  The tier cap the dispatcher leaves in
 * the flags' CPU field is not a device ordinal: cleared. */
#define QS_TIER(name) JPEGQS_ATTR int do_quantsmooth_##name(j_decompress_ptr srcinfo, jvirt_barray_ptr *coef_arrays, \
		jpegqs_control_t *opts) { \
	jpegqs_control_t o = *opts; \
	o.flags &= ~(JPEGQS_CPU_MASK << JPEGQS_CPU_SHIFT); \
	return do_quantsmooth(srcinfo, coef_arrays, &o); }
QS_TIER(base) QS_TIER(sse2) QS_TIER(avx2) QS_TIER(avx512)

#ifndef TRANSCODE_ONLY
/* decode helpers, reference quantsmooth.h:2880-2904: read every scan in buffered-image
 * mode, smooth the coefficient arrays, then let the caller pull scanlines as usual */
JPEGQS_ATTR
boolean jpegqs_start_decompress(j_decompress_ptr cinfo, jpegqs_control_t *opts) {
	boolean ok;
	int active = opts->niter > 0 || (opts->flags & JPEGQS_UPSAMPLE_UV);
	if (!jpeg_start_decompress || !jpeg_input_complete || !jpeg_start_output || !jpeg_finish_output ||
			!jpeg_read_coefficients) {
		fprintf(stderr, "jpegqs: jpegqs_start_decompress needs libjpeg loaded in this process\n");
		return FALSE;
	}
	if (active) cinfo->buffered_image = TRUE;
	ok = jpeg_start_decompress(cinfo);
	if (!active) return ok;
	while (!jpeg_input_complete(cinfo)) {
		jpeg_start_output(cinfo, cinfo->input_scan_number);
		jpeg_finish_output(cinfo);
	}
	do_quantsmooth(cinfo, jpeg_read_coefficients(cinfo), opts);
	jpeg_start_output(cinfo, cinfo->input_scan_number);
	return ok;
}

JPEGQS_ATTR
boolean jpegqs_finish_decompress(j_decompress_ptr cinfo) {
	if (!jpeg_finish_output || !jpeg_finish_decompress) return FALSE;
	if (cinfo->buffered_image &&
			(cinfo->global_state == DSTATE_SCANNING || cinfo->global_state == DSTATE_RAW_OK))
		jpeg_finish_output(cinfo);
	return jpeg_finish_decompress(cinfo);
}
#endif
