/*
 * qs_compress.cu - jpegqs_cuda_compress_async: 8-bit pictures in device memory to the JPEG files
 * Pillow's Image.save(quality, subsampling, optimize) writes for them, and jpegqs_cuda_compress_model,
 * the same steps on one CPU thread.  DESIGN.md section 3.11 describes the scheme; in short:
 *
 *   front half  one launch per group of pictures turns every component of every picture into quantized
 *               coefficients in libjpeg's block layout ([hblk][wblk][64], natural order).  One thread
 *               makes one 8x8 block: it reads the full-resolution pixels the block's samples come from,
 *               converts them to the component (jccolor.c rgb_ycc_convert, or a copy for grey),
 *               down-samples them (jcsample.c fullsize / h2v1 / h2v2, with libjpeg's edge rules), runs
 *               jfdctint.c's jpeg_fdct_islow and quantizes (jcdctmgr.c).  A CTA finds its component by
 *               a binary search over the components' first CTAs, as qs_resize.cu's passes do.
 *   back half   jpegqs_cuda_encode_async over those coefficients with the quality-scaled tables and the
 *               JFIF prefix libjpeg writes, which the compressor kernel copies from its parameters into
 *               the workspace.
 *
 * libjpeg-turbo's compressor writes the same bytes with and without its SIMD code, so its C code
 * (jccolor.c, jcsample.c, jcprepct.c, jfdctint.c, jcdctmgr.c) is what this restates, integer for integer.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <memory>
#include <vector>
#include "../../include/jpegqs_cuda.h"

#define HD __host__ __device__
#define QC_THREADS 128                 /* blocks per CTA: one thread each                        */
#define QC_PACK 32                     /* pictures per launch group (three components each)      */
#define QC_PREFIX_LEN 20               /* SOI + JFIF APP0                                        */

/* SOI and the JFIF 1.01 APP0 libjpeg writes with Pillow's defaults: density unit 0, 1:1, no thumbnail */
static const uint8_t qc_prefix[QC_PREFIX_LEN] = {
	0xFF, 0xD8, 0xFF, 0xE0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0x00, 0x01, 0x01, 0x00, 0x00, 0x01, 0x00, 0x01, 0x00, 0x00 };

/* jcparam.c's base tables (T.81 K.1), natural order */
static const uint8_t qc_std_luma[64] = {
	16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
	14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
	49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99 };
static const uint8_t qc_std_chroma[64] = {
	17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
	47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
	99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99 };

/* ---------------------------------------------------------------- one component of one picture */
struct QcJob {
	const uint8_t *src;                /* the picture, HWC                                        */
	uint64_t row_bytes;
	int16_t *coef;                     /* [hblk][wblk][64]                                        */
	uint32_t first;                    /* its first CTA in the launch                             */
	uint32_t width, height;            /* the picture                                             */
	uint32_t wblk, hblk;
	uint32_t dh;                       /* downsampled_height: rows past it repeat its last row    */
	uint8_t ch, comp, sx, sy;          /* channels; component 0..2; down-sampling factors 1 or 2  */
	uint16_t q[64];                    /* quantization table, natural order                       */
};

/* ---------------------------------------------------------------- the arithmetic, host and device */
#define QC_SCALEBITS 16
#define QC_FIX(x) ((int32_t)((x) * (1L << QC_SCALEBITS) + 0.5))
#define QC_ONE_HALF ((int32_t)1 << (QC_SCALEBITS - 1))
#define QC_CBCR_OFFSET ((int32_t)128 << QC_SCALEBITS)

/* component `comp` of the full-resolution pixel (x, y), inside the picture: rgb_ycc_convert's sums */
HD static inline int qc_pixel(const QcJob &j, uint32_t x, uint32_t y) {
	const uint8_t *p = j.src + (size_t)y * j.row_bytes + (size_t)x * j.ch;
	if (j.ch == 1) return p[0];
	const int32_t r = p[0], g = p[1], b = p[2];
	if (j.comp == 0)
		return (int)((QC_FIX(0.29900) * r + QC_FIX(0.58700) * g + QC_FIX(0.11400) * b + QC_ONE_HALF) >> QC_SCALEBITS);
	if (j.comp == 1)
		return (int)((-QC_FIX(0.16874) * r - QC_FIX(0.33126) * g + QC_FIX(0.50000) * b + QC_CBCR_OFFSET + QC_ONE_HALF - 1) >> QC_SCALEBITS);
	return (int)((QC_FIX(0.50000) * r - QC_FIX(0.41869) * g - QC_FIX(0.08131) * b + QC_CBCR_OFFSET + QC_ONE_HALF - 1) >> QC_SCALEBITS);
}

/* down-sampled sample (cx, cy) of the component, anywhere in its blocks.
 *   right edge   expand_right_edge runs on the full-resolution rows before down-sampling: columns
 *                past the picture repeat column width - 1;
 *   bottom edge  jcprepct.c repeats the last full-resolution row inside the last row group, down-samples,
 *                then repeats the last down-sampled row (dh - 1) down to the block rows' end.
 * h2v1 adds a bias of 0, 1, 0, 1, ... per output column, h2v2 1, 2, 1, 2, ... (jcsample.c). */
HD static inline int qc_sample(const QcJob &j, uint32_t cx, uint32_t cy) {
	if (cy >= j.dh) cy = j.dh - 1;
	const uint32_t xm = j.width - 1, ym = j.height - 1;
	uint32_t x0 = cx * j.sx, y0 = cy * j.sy;
	const uint32_t x1 = x0 + 1 < xm ? x0 + 1 : xm, y1 = y0 + 1 < ym ? y0 + 1 : ym;
	x0 = x0 < xm ? x0 : xm; y0 = y0 < ym ? y0 : ym;
	if (j.sx == 1) return qc_pixel(j, x0, y0);
	if (j.sy == 1) return (qc_pixel(j, x0, y0) + qc_pixel(j, x1, y0) + (int)(cx & 1)) >> 1;
	return (qc_pixel(j, x0, y0) + qc_pixel(j, x1, y0) + qc_pixel(j, x0, y1) + qc_pixel(j, x1, y1) + 1 + (int)(cx & 1)) >> 2;
}

/* jfdctint.c's jpeg_fdct_islow: CONST_BITS 13, PASS1_BITS 2, output scaled up by 8 */
#define QC_CB 13
#define QC_P1 2
#define QC_DESCALE(x, n) (((x) + ((int32_t)1 << ((n) - 1))) >> (n))
HD static inline void qc_fdct_1d(int32_t *d, int s, bool pass1) {
	const int32_t tmp0 = d[0] + d[7 * s], tmp7 = d[0] - d[7 * s];
	const int32_t tmp1 = d[s] + d[6 * s], tmp6 = d[s] - d[6 * s];
	const int32_t tmp2 = d[2 * s] + d[5 * s], tmp5 = d[2 * s] - d[5 * s];
	const int32_t tmp3 = d[3 * s] + d[4 * s], tmp4 = d[3 * s] - d[4 * s];
	const int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
	const int sh = pass1 ? QC_CB - QC_P1 : QC_CB + QC_P1;
	if (pass1) { d[0] = (tmp10 + tmp11) << QC_P1; d[4 * s] = (tmp10 - tmp11) << QC_P1; }
	else { d[0] = QC_DESCALE(tmp10 + tmp11, QC_P1); d[4 * s] = QC_DESCALE(tmp10 - tmp11, QC_P1); }
	const int32_t z1 = (tmp12 + tmp13) * 4433;                          /* FIX_0_541196100 */
	d[2 * s] = QC_DESCALE(z1 + tmp13 * 6270, sh);                       /* FIX_0_765366865 */
	d[6 * s] = QC_DESCALE(z1 - tmp12 * 15137, sh);                      /* FIX_1_847759065 */
	const int32_t z5 = (tmp4 + tmp5 + tmp6 + tmp7) * 9633;              /* FIX_1_175875602 */
	const int32_t a4 = tmp4 * 2446, a5 = tmp5 * 16819, a6 = tmp6 * 25172, a7 = tmp7 * 12299;
	const int32_t z1o = -(tmp4 + tmp7) * 7373, z2 = -(tmp5 + tmp6) * 20995;
	const int32_t z3 = -(tmp4 + tmp6) * 16069 + z5, z4 = -(tmp5 + tmp7) * 3196 + z5;
	d[7 * s] = QC_DESCALE(a4 + z1o + z3, sh);
	d[5 * s] = QC_DESCALE(a5 + z2 + z4, sh);
	d[3 * s] = QC_DESCALE(a6 + z2 + z3, sh);
	d[s] = QC_DESCALE(a7 + z1o + z4, sh);
}

/* jcdctmgr.c's quantization of an islow output: divisor 8 * q, rounded half away from zero */
HD static inline int16_t qc_quant(int32_t t, int32_t q) {
	const int32_t q8 = q << 3, a = t < 0 ? -t : t, v = (a + (q8 >> 1)) / q8;
	return (int16_t)(t < 0 ? -v : v);
}

/* block (bx, by) of the component: 64 quantized coefficients, natural order */
HD static inline void qc_block(const QcJob &j, uint32_t bx, uint32_t by, int16_t *out) {
	int32_t d[64];
#pragma unroll
	for (int y = 0; y < 8; y++)
#pragma unroll
		for (int x = 0; x < 8; x++) d[8 * y + x] = qc_sample(j, 8 * bx + x, 8 * by + y) - 128;
#pragma unroll
	for (int y = 0; y < 8; y++) qc_fdct_1d(d + 8 * y, 1, true);
#pragma unroll
	for (int x = 0; x < 8; x++) qc_fdct_1d(d + x, 8, false);
#pragma unroll
	for (int k = 0; k < 64; k++) out[k] = qc_quant(d[k], j.q[k]);
}

/* ---------------------------------------------------------------- the kernel */
struct QcPack {
	QcJob job[3 * QC_PACK];
	int njob;
	uint8_t *prefix_dev;               /* where the JFIF prefix goes (the workspace)               */
	uint8_t prefix[QC_PREFIX_LEN];
};
static_assert(sizeof(QcPack) <= 32000, "QcPack exceeds the kernel parameter space");

__global__ void __launch_bounds__(QC_THREADS) qc_compress_kernel(const __grid_constant__ QcPack P) {
	if (blockIdx.x == 0 && threadIdx.x < QC_PREFIX_LEN) P.prefix_dev[threadIdx.x] = P.prefix[threadIdx.x];
	int lo = 0, hi = P.njob - 1;                        /* the last component whose first CTA is <= this one */
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (P.job[mid].first <= blockIdx.x) lo = mid; else hi = mid - 1;
	}
	const QcJob &j = P.job[lo];
	const uint32_t b = (blockIdx.x - j.first) * QC_THREADS + threadIdx.x;
	if (b >= j.wblk * j.hblk) return;
	const uint32_t by = b / j.wblk, bx = b - by * j.wblk;
	__align__(16) int16_t blk[64];
	qc_block(j, bx, by, blk);
	int4 *dst = reinterpret_cast<int4 *>(j.coef + (size_t)b * 64);
	const int4 *s = reinterpret_cast<const int4 *>(blk);
#pragma unroll
	for (int k = 0; k < 8; k++) dst[k] = s[k];
}

/* Pillow sets the luma sampling factors whatever the component count, so a grey file's SOF says 2x1
 * or 2x2 under 4:2:2 or 4:2:0.  libjpeg codes a single-component scan block by block all the same, so
 * the encoder is given 1x1 and this byte (the component's sampling in SOF, after the 20-byte prefix and
 * the 69-byte DQT) is set afterwards, inside the capacity. */
#define QC_GREY_SOF_SAMP 100
struct QcGreyFix { uint8_t *out[QC_PACK]; uint64_t cap[QC_PACK]; int n; uint8_t samp; };
__global__ void qc_grey_fix_kernel(const __grid_constant__ QcGreyFix F) {
	const int i = threadIdx.x;
	if (i < F.n && F.cap[i] > QC_GREY_SOF_SAMP) F.out[i][QC_GREY_SOF_SAMP] = F.samp;
}

/* ---------------------------------------------------------------- host: geometry, checks, sizes */
struct jpegqs_cuda_ctx;
void qs_ctx_decode_info(jpegqs_cuda_ctx *ctx, int *device, cudaStream_t *stream, int *sub_bytes);
void qs_ctx_decode_done(jpegqs_cuda_ctx *ctx, int launches, const char *err);
extern "C" void qs_set_host_error(const char *msg);

static size_t qc_a256(size_t x) { return (x + 255) & ~(size_t)255; }

static const char *qc_check_params(const jpegqs_cuda_jpeg_params *jp) {
	if (!jp) return "params NULL";
	if (jp->quality < 1 || jp->quality > 100) return "quality outside 1..100";
	if (jp->subsampling < 0 || jp->subsampling > 2) return "subsampling outside 0..2";
	if ((jp->optimize & ~(JPEGQS_JPEG_PROGRESSIVE | 1)) != 0) return "optimize other than 0 / 1, ORed with JPEGQS_JPEG_PROGRESSIVE";
	return NULL;
}

/* jpeg_set_quality(quality, force_baseline = TRUE): table `which` (0 luma, 1 chroma), natural order */
static void qc_table(int quality, int which, uint16_t *q) {
	const int scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
	const uint8_t *base = which ? qc_std_chroma : qc_std_luma;
	for (int i = 0; i < 64; i++) {
		long t = ((long)base[i] * scale + 50) / 100;
		q[i] = (uint16_t)(t < 1 ? 1 : t > 255 ? 255 : t);
	}
}

/* the encoder's image for a picture (coefficient pointers NULL) and its components' jobs (src, coef
 * and first unset); returns NULL or what is wrong with the picture */
static const char *qc_geometry(const jpegqs_cuda_pixels_in &p, const jpegqs_cuda_jpeg_params &jp, jpegqs_cuda_image *im,
		QcJob *jobs) {
	if (p.width < 1 || p.width > 65535 || p.height < 1 || p.height > 65535) return "picture size outside 1..65535";
	if (p.channels != 1 && p.channels != 3) return "channels other than 1 or 3";
	if (p.row_bytes < (size_t)p.width * p.channels) return "row_bytes smaller than width * channels";
	memset(im, 0, sizeof(*im));
	const int nc = p.channels;
	const int lh = nc == 3 && jp.subsampling ? 2 : 1, lv = nc == 3 && jp.subsampling == 2 ? 2 : 1;
	/* is_ycbcr 0: the encoder's up-sampled geometry (UPSAMPLE_UV) never applies here, and its bound and
	 * workspace then cover the sampled geometry only */
	im->ncomp = nc; im->is_ycbcr = 0; im->image_width = (uint32_t)p.width; im->image_height = (uint32_t)p.height;
	for (int c = 0; c < nc; c++) {
		jpegqs_cuda_comp &cc = im->comp[c];
		cc.h_samp = c ? 1 : lh; cc.v_samp = c ? 1 : lv; cc.has_qtbl = 1;
		const uint32_t dw = (uint32_t)(((uint64_t)p.width * cc.h_samp + lh - 1) / lh);
		const uint32_t dh = (uint32_t)(((uint64_t)p.height * cc.v_samp + lv - 1) / lv);
		cc.wblk = (dw + 7) / 8; cc.hblk = (dh + 7) / 8;
		qc_table(jp.quality, c ? 1 : 0, cc.quant);
		QcJob &j = jobs[c];
		memset(&j, 0, sizeof(j));
		j.row_bytes = p.row_bytes; j.width = (uint32_t)p.width; j.height = (uint32_t)p.height;
		j.wblk = cc.wblk; j.hblk = cc.hblk; j.dh = dh;
		j.ch = (uint8_t)nc; j.comp = (uint8_t)c; j.sx = (uint8_t)(lh / cc.h_samp); j.sy = (uint8_t)(lv / cc.v_samp);
		memcpy(j.q, cc.quant, sizeof(j.q));
	}
	return NULL;
}

/* the SOF sampling byte Pillow's settings give a grey file */
static uint8_t qc_grey_samp(const jpegqs_cuda_jpeg_params &jp) { return jp.subsampling == 2 ? 0x22 : jp.subsampling == 1 ? 0x21 : 0x11; }

static jpegqs_cuda_jpeg_head qc_head(const uint8_t *prefix, int nc) {
	jpegqs_cuda_jpeg_head h;
	memset(&h, 0, sizeof(h));
	h.prefix_dev = prefix; h.prefix_len = QC_PREFIX_LEN;
	for (int c = 0; c < nc; c++) { h.comp_id[c] = c + 1; h.quant_tbl[c] = c ? 1 : 0; }
	return h;
}

/* the progressive coder of qs_encode.cu */
size_t qe_progressive_bound(const jpegqs_cuda_image *img, size_t prefix_len);
size_t qe_progressive_workspace(const jpegqs_cuda_image *img);
int qe_progressive_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_image *imgs, const jpegqs_cuda_jpeg_head *heads,
		uint8_t *const *out_dev, const size_t *out_cap, uint64_t *len_dev, int32_t *status_dev, void *workspace,
		size_t workspace_bytes, cudaStream_t st);
int qe_progressive_model(const jpegqs_cuda_image *img, const jpegqs_cuda_jpeg_head *head, uint8_t *out, size_t cap,
		uint64_t *len, int32_t *status);

static bool qc_progressive(const jpegqs_cuda_jpeg_params &jp) { return (jp.optimize & JPEGQS_JPEG_PROGRESSIVE) != 0; }

static size_t qc_coef_bytes(const jpegqs_cuda_image &im) {
	size_t b = 0;
	for (int c = 0; c < im.ncomp; c++) b += qc_a256((size_t)im.comp[c].wblk * im.comp[c].hblk * 128);
	return b;
}

extern "C" int jpegqs_cuda_compress_bound(const jpegqs_cuda_pixels_in *pic, const jpegqs_cuda_jpeg_params *params, size_t *bytes) {
	char m[256];
	const char *e = !pic || !bytes ? "NULL argument" : qc_check_params(params);
	jpegqs_cuda_image im; QcJob jobs[3];
	if (!e) e = qc_geometry(*pic, *params, &im, jobs);
	if (e) { snprintf(m, sizeof(m), "jpegqs_cuda_compress_bound: %s", e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
	if (qc_progressive(*params)) { *bytes = qe_progressive_bound(&im, QC_PREFIX_LEN); return 0; }
	return jpegqs_cuda_encode_bound(&im, QC_PREFIX_LEN, bytes);
}

/* one picture's share of the workspace: its coefficients and its encoder workspace */
static int qc_share(const jpegqs_cuda_image &im, int optimize, size_t *bytes) {
	size_t w = 0;
	int r = 0;
	if (optimize & JPEGQS_JPEG_PROGRESSIVE) w = qe_progressive_workspace(&im);
	else r = jpegqs_cuda_encode_workspace_bytes(1, &im, optimize, &w);
	*bytes = qc_coef_bytes(im) + w;
	return r;
}

extern "C" int jpegqs_cuda_compress_workspace_bytes(int n, const jpegqs_cuda_pixels_in *pics, const jpegqs_cuda_jpeg_params *params,
		size_t *bytes) {
	char m[256];
	const char *e = n < 0 || !bytes || (n && !pics) ? "NULL argument" : qc_check_params(params);
	if (e) { snprintf(m, sizeof(m), "jpegqs_cuda_compress_workspace_bytes: %s", e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
	size_t total = 256;                                  /* the prefix */
	for (int i = 0; i < n; i++) {
		jpegqs_cuda_image im; QcJob jobs[3]; size_t b;
		if ((e = qc_geometry(pics[i], *params, &im, jobs))) {
			snprintf(m, sizeof(m), "jpegqs_cuda_compress_workspace_bytes: picture %d: %s", i, e); qs_set_host_error(m); return JPEGQS_ERR_ARG;
		}
		int r = qc_share(im, params->optimize, &b);
		if (r < 0) return r;
		total += b;
	}
	*bytes = total;
	return 0;
}

#define QC_CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	snprintf(msg, sizeof(msg), "%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
	qs_ctx_decode_done(ctx, launches, msg); return JPEGQS_ERR_CUDA; } } while (0)

extern "C" int jpegqs_cuda_compress_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_pixels_in *pics,
		const jpegqs_cuda_jpeg_params *params, uint8_t *const *out_dev, const size_t *out_cap, uint64_t *len_dev,
		int32_t *status_dev, void *workspace, size_t workspace_bytes, void *stream) {
	char msg[512] = "";
	int launches = 0;
	if (!ctx) return JPEGQS_ERR_ARG;
	int device, unused; cudaStream_t st;
	qs_ctx_decode_info(ctx, &device, &st, &unused);
	if (stream) st = (cudaStream_t)stream;
	if (n < 0 || (n && (!pics || !out_dev || !out_cap || !len_dev || !status_dev || !workspace))) {
		qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_compress_async: NULL argument"); return JPEGQS_ERR_ARG;
	}
	const char *e = qc_check_params(params);
	if (e) { snprintf(msg, sizeof(msg), "jpegqs_cuda_compress_async: %s", e); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
	if ((uintptr_t)workspace & 255) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_compress_async: workspace not 256-byte aligned"); return JPEGQS_ERR_ARG; }
	std::vector<jpegqs_cuda_image> imgs((size_t)n);
	std::vector<QcJob> jobs(3 * (size_t)n);
	std::vector<size_t> share((size_t)n);
	size_t need = 256;
	for (int i = 0; i < n; i++) {
		e = qc_geometry(pics[i], *params, &imgs[i], &jobs[3 * i]);
		if (!e && !pics[i].pixels_dev) e = "pixels_dev NULL";
		if (!e && !out_dev[i]) e = "out_dev entry NULL";
		if (!e && out_cap[i] < QC_PREFIX_LEN) e = "out_cap smaller than the 20-byte prefix";
		if (e) { snprintf(msg, sizeof(msg), "jpegqs_cuda_compress_async: picture %d: %s", i, e); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
		int r = qc_share(imgs[i], params->optimize, &share[i]);
		if (r < 0) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_compress_async: encoder geometry"); return r; }
		need += share[i];
	}
	if (workspace_bytes < need) {
		snprintf(msg, sizeof(msg), "jpegqs_cuda_compress_async: workspace of %zu bytes, %zu needed", workspace_bytes, need);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (!n) { qs_ctx_decode_done(ctx, 0, ""); return 0; }
	QC_CK(cudaSetDevice(device));
	/* workspace: the prefix, then every picture's coefficients, then the encoder's workspace */
	char *w = (char *)workspace;
	uint8_t *prefix = (uint8_t *)w;
	w += 256;
	for (int i = 0; i < n; i++)
		for (int c = 0; c < imgs[i].ncomp; c++) {
			jpegqs_cuda_comp &cc = imgs[i].comp[c];
			cc.coef = (int16_t *)w; w += qc_a256((size_t)cc.wblk * cc.hblk * 128);
			QcJob &j = jobs[3 * i + c];
			j.src = pics[i].pixels_dev; j.coef = cc.coef;
		}
	const size_t ws_enc = workspace_bytes - (size_t)(w - (char *)workspace);
	std::unique_ptr<QcPack> hold(new QcPack());          /* ~20 KB: not on the stack */
	QcPack &P = *hold;
	for (int g0 = 0; g0 < n; g0 += QC_PACK) {
		const int g = n - g0 < QC_PACK ? n - g0 : QC_PACK;
		memset(&P, 0, sizeof(P));
		P.prefix_dev = prefix;
		memcpy(P.prefix, qc_prefix, QC_PREFIX_LEN);
		uint64_t ctas = 0;
		for (int i = g0; i < g0 + g; i++)
			for (int c = 0; c < imgs[i].ncomp; c++) {
				QcJob j = jobs[3 * i + c];
				j.first = (uint32_t)ctas;
				ctas += ((uint64_t)j.wblk * j.hblk + QC_THREADS - 1) / QC_THREADS;
				P.job[P.njob++] = j;
			}
		if (ctas > 0x7FFFFFFFull) { qs_ctx_decode_done(ctx, launches, "jpegqs_cuda_compress_async: pictures too large"); return JPEGQS_ERR_ARG; }
		qc_compress_kernel<<<(unsigned)ctas, QC_THREADS, 0, st>>>(P); launches++;
		QC_CK(cudaGetLastError());
	}
	std::vector<jpegqs_cuda_jpeg_head> heads((size_t)n);
	for (int i = 0; i < n; i++) heads[i] = qc_head(prefix, imgs[i].ncomp);
	int r = qc_progressive(*params)
		? qe_progressive_async(ctx, n, imgs.data(), heads.data(), out_dev, out_cap, len_dev, status_dev, w, ws_enc, st)
		: jpegqs_cuda_encode_async(ctx, n, imgs.data(), heads.data(), params->optimize, NULL, out_dev, out_cap, len_dev,
			status_dev, w, ws_enc, st);
	if (r < 0) return r;
	launches += jpegqs_cuda_last_launches(ctx);
	if (params->subsampling) {
		QcGreyFix F;
		memset(&F, 0, sizeof(F));
		F.samp = qc_grey_samp(*params);
		for (int i = 0; i <= n; i++) {
			if (i == n || F.n == QC_PACK) {
				if (F.n) { qc_grey_fix_kernel<<<1, QC_PACK, 0, st>>>(F); launches++; QC_CK(cudaGetLastError()); }
				F.n = 0;
			}
			if (i < n && pics[i].channels == 1) { F.out[F.n] = out_dev[i]; F.cap[F.n] = out_cap[i]; F.n++; }
		}
	}
	qs_ctx_decode_done(ctx, launches, "");
	return 0;
}

/* ---------------------------------------------------------------- the CPU model */
extern "C" int jpegqs_cuda_compress_model(const jpegqs_cuda_pixels_in *pic, const jpegqs_cuda_jpeg_params *params,
		uint8_t *out, size_t cap, uint64_t *len, int32_t *status) {
	char m[256];
	jpegqs_cuda_image im; QcJob jobs[3];
	const char *e = !pic || !out || !len || !status ? "NULL argument" : qc_check_params(params);
	if (!e) e = qc_geometry(*pic, *params, &im, jobs);
	if (!e && !pic->pixels_dev) e = "pixels NULL";
	if (!e && cap < QC_PREFIX_LEN) e = "cap smaller than the 20-byte prefix";
	if (e) { snprintf(m, sizeof(m), "jpegqs_cuda_compress_model: %s", e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
	std::vector<int16_t> coef[3];
	for (int c = 0; c < im.ncomp; c++) {
		QcJob &j = jobs[c];
		coef[c].assign((size_t)j.wblk * j.hblk * 64, 0);
		j.src = pic->pixels_dev; j.coef = coef[c].data();
		im.comp[c].coef = coef[c].data();
		for (uint32_t by = 0; by < j.hblk; by++)
			for (uint32_t bx = 0; bx < j.wblk; bx++) qc_block(j, bx, by, j.coef + ((size_t)by * j.wblk + bx) * 64);
	}
	jpegqs_cuda_jpeg_head h = qc_head(qc_prefix, im.ncomp);
	int r = qc_progressive(*params) ? qe_progressive_model(&im, &h, out, cap, len, status)
		: jpegqs_cuda_encode_model(&im, &h, params->optimize, out, cap, len, status);
	if (!r && im.ncomp == 1 && params->subsampling && cap > QC_GREY_SOF_SAMP) out[QC_GREY_SOF_SAMP] = qc_grey_samp(*params);
	return r;
}
