/*
 * libjpegqs.h - public API of the H100-native (sm_90a) quantsmooth library.
 *
 * Source compatible with the reference's API header (reference libjpegqs.h:14-55): the same
 * identifiers with the same values, the same jpegqs_control_t layout and the same three entry
 * points.  A caller that includes "libjpegqs.h" (irfanview/plugin.c, and quantsmooth.c in its
 * SIMD_SELECT build, which includes libjpegqs.c -> libjpegqs.h) compiles against this header and
 * links against libjpegqs_b200.so as is; quantsmooth.c:89 and example.c:37 include the
 * implementation header "quantsmooth.h" instead and need that one line changed to "libjpegqs.h"
 * (example.c:36 says so itself).  INTEGRATION.md section 2 has the build lines that were run.
 * Include <jpeglib.h> before this header.
 *
 * Behavioural differences (INTEGRATION.md):
 *   - the smoothing runs on a CUDA device (sm_90a).  There is no CPU fallback: without a
 *     usable device do_quantsmooth reports on stderr and returns a negative value, leaving
 *     the coefficients untouched;
 *   - jpegqs_control_t.threads is ignored (reference: OpenMP thread count,
 *     quantsmooth.h:2467-2472);
 *   - (flags >> JPEGQS_CPU_SHIFT) & JPEGQS_CPU_MASK selects the CUDA device ordinal + 1
 *     (0 = current device) instead of capping the SIMD tier (reference libjpegqs.c:123-129).
 */
#ifndef JPEGQS_B200_LIBJPEGQS_H
#define JPEGQS_B200_LIBJPEGQS_H
#ifndef JPEGQS_H
#define JPEGQS_H                       /* the reference's guard: both headers exclude each other */
#endif

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* behaviour flags, jpegqs_control_t.flags bits 0..6 */
enum jpegqs_flag_bits {
	JPEGQS_DIAGONALS       = 1 << 0,   /* -q >= 4: add the 98 diagonal pixel pairs             */
	JPEGQS_JOINT_YUV       = 1 << 1,   /* -q >= 5: predict chroma from the smoothed luma        */
	JPEGQS_UPSAMPLE_UV     = 1 << 2,   /* -q >= 6: re-sample sub-sampled chroma at luma size     */
	JPEGQS_LOW_QUALITY     = 1 << 3,   /* -q <= 2: one-shot 8-neighbour filter                   */
	JPEGQS_NO_REBALANCE    = 1 << 4,
	JPEGQS_NO_REBALANCE_UV = 1 << 5,
	JPEGQS_TRANSCODE       = 1 << 6,   /* caller re-encodes the coefficients (no decoder re-init) */
	JPEGQS_FLAGS_MASK      = 0x7f
};

/* bit fields above the behaviour flags */
enum jpegqs_flag_fields {
	JPEGQS_CPU_SHIFT  = 12,            /* 4 bits: here the CUDA device ordinal + 1               */
	JPEGQS_CPU_MASK   = 15,
	JPEGQS_INFO_SHIFT = 16             /* log selection, JPEGQS_INFO_* below                     */
};

enum jpegqs_info_bits {
	JPEGQS_INFO_COMP1 = 1 << 16,       /* component sampling factors and table numbers           */
	JPEGQS_INFO_QUANT = 1 << 17,       /* quantization tables                                    */
	JPEGQS_INFO_COMP2 = 1 << 18,       /* component sizes in blocks                              */
	JPEGQS_INFO_TIME  = 1 << 19,       /* "quantsmooth: %.3fms"                                  */
	JPEGQS_INFO_CPU   = 1 << 20        /* back end report ("SIMD type: ...")                     */
};

enum jpegqs_limits { JPEGQS_ITER_MAX = 100 };   /* niter is clamped to [0, JPEGQS_ITER_MAX] */

#ifndef JPEGQS_ATTR
#define JPEGQS_ATTR
#endif

#define JPEGQS_VERSION "1.20230818-b200"
/* the reference CLI prints this next to the version (quantsmooth.c:472); the algorithm is its
 * author's, the sm_90a back end is this repository's */
#define JPEGQS_COPYRIGHT "algorithm (C) 2020-2026 Ilya Kurdyukov, CUDA back end (C) 2026 jpeg-quantsmooth_b200"

typedef struct jpegqs_control {
	int flags;                         /* JPEGQS_* bits                                          */
	int niter;                         /* iterations                                             */
	int threads;                       /* ignored by this back end                               */
	int progprec;                      /* number of progress steps (0 = 20, < 0 = every row unit)   */
	void *userdata;                    /* passed to progress()                                   */
	int (*progress)(void *data, int cur, int max);   /* non-zero return = stop                 */
} jpegqs_control_t;

/* smooths the coefficient arrays in place; replaces reference libjpegqs.h:47-48 / quantsmooth.h:2404 */
JPEGQS_ATTR int do_quantsmooth(j_decompress_ptr srcinfo, jvirt_barray_ptr *coef_arrays,
		jpegqs_control_t *opts);

/* extension: create the CUDA context do_quantsmooth(flags) will use (device from the CPU field),
 * e.g. on a second thread while the caller still decodes its file; returns 0 or a negative value */
JPEGQS_ATTR int jpegqs_warmup(int flags);

/* extension: one JPEG file in memory to the file that reading it, do_quantsmooth(opts) and writing it
 * (optimize, copy: the jpegqs tool's -o and -c) give, byte for byte, with the same -i lines on stderr -
 * decoded, smoothed and encoded on the device do_quantsmooth(opts) uses (include/jpegqs_cuda.h
 * jpegqs_cuda_transcode).  Returns 0 (*out: the file, malloc'd), 1 when the caller must take its
 * own route for this file (nothing printed; *reason, a static string, says why: damaged data, a file
 * the device route does not take) or a negative value, reported on stderr as do_quantsmooth does. */
JPEGQS_ATTR int jpegqs_transcode(const unsigned char *data, size_t len, int copy, int optimize,
		jpegqs_control_t *opts, unsigned char **out, size_t *outlen, const char **reason);
/* extension: jpegqs_transcode for n files in shared device launches (jpegqs_cuda_transcode_batch).
 * rc[i], out[i], outlen[i] and reason[i] are what jpegqs_transcode returns for file i alone.  Each
 * file's -i lines and error messages are those of jpegqs_transcode; a file's time line shows the wall
 * time of the whole call.  log NULL: they reach stderr, file by file in their order; otherwise log[i]
 * receives file i's text (malloc'd, NULL when there is none, always NULL for a file that falls back)
 * for the caller to print and free - so a caller can print them in order with the host route's
 * output for the files that fall back.  Returns 0. */
JPEGQS_ATTR int jpegqs_transcode_batch(int n, const unsigned char *const *data, const size_t *len, int copy,
		int optimize, jpegqs_control_t *opts, unsigned char **out, size_t *outlen, int *rc, const char **reason,
		char **log);

#ifndef TRANSCODE_ONLY
/* decode helpers; replace reference libjpegqs.h:50-55 / quantsmooth.h:2880-2904 */
JPEGQS_ATTR boolean jpegqs_start_decompress(j_decompress_ptr cinfo, jpegqs_control_t *opts);
JPEGQS_ATTR boolean jpegqs_finish_decompress(j_decompress_ptr cinfo);
#endif

#ifdef __cplusplus
}
#endif
#endif
