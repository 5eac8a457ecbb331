/*
 * qs_reduce.cu - reduce 8-bit pictures by integer factors exactly as Pillow's Image.reduce does
 * (libImaging/Reduce.c): the reduce stage of jpegqs_cuda_pixels_batch_reduced, which Pillow's
 * Image.resize(..., reducing_gap=) and Image.thumbnail run before the resize, and
 * jpegqs_cuda_reduce_model, the same computation on one CPU thread.  Also the host planning of those
 * two calls (_get_safe_box, the shifted float box, thumbnail's size and draft scale) and
 * jpegqs_cuda_thumbnail_geometry / jpegqs_cuda_resize_model_box on top of it.
 *
 * Reduce.c sums each cell of fx x fy samples (fewer at the right and bottom edges of the box) in 32-bit
 * unsigned arithmetic and divides by multiplication: ((sum + n / 2) * m) >> 24 with
 * m = (uint32)((float)2^32 / (float)(256 * n)), n the cell's sample count.  That is not the rounded mean;
 * it is restated here operation for operation.  The sum is an integer sum, so the order of the taps
 * does not matter.
 *
 * One launch reduces every picture of a sub-batch.  A block takes up to QS_RD_THREADS consecutive bytes
 * of one output row, one byte (one cell of one channel) per thread, and finds its picture by a binary
 * search over the pictures' first blocks, as the resize kernels do.  The tap loops have no fixed bound.
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <vector>
#include "qs_reduce.h"

extern "C" void qs_set_host_error(const char *msg);        /* qs_cuda.cu: jpegqs_cuda_last_error(NULL) */

#define QS_RD_THREADS 256

/* ---- the per-sample arithmetic (device and host model) -------------------------------------------- */
/* Reduce.c's division_UINT32(n, 8): 2^32 as a float over the int 256 * n converted to float */
__host__ __device__ static inline uint32_t qs_rd_multiplier(uint32_t n) {
	const float dividend = (float)(256u * n);
#ifdef __CUDA_ARCH__
	return (uint32_t)__fdiv_rn(4294967296.0f, dividend);
#else
	return (uint32_t)(4294967296.0f / dividend);
#endif
}

/* byte j of output row y */
__host__ __device__ static inline uint8_t qs_rd_sample(const QsReduceDesc &d, uint32_t y, uint32_t j) {
	const uint32_t x = j / d.ch, c = j - x * d.ch;
	const int32_t x0 = (int32_t)x * d.fx, y0 = (int32_t)y * d.fy;
	const int32_t nx = d.box_w - x0 < d.fx ? d.box_w - x0 : d.fx, ny = d.box_h - y0 < d.fy ? d.box_h - y0 : d.fy;
	const uint32_t n = (uint32_t)nx * (uint32_t)ny;
	const size_t stride = (size_t)d.src_w * d.ch;
	const uint8_t *s = d.src + (size_t)(d.top + y0) * stride + ((size_t)d.left + x0) * d.ch + c;
	uint32_t ss = n / 2;
	for (int32_t yy = 0; yy < ny; yy++, s += stride)
		for (int32_t xx = 0; xx < nx; xx++) ss += s[(size_t)xx * d.ch];
	return (uint8_t)((ss * qs_rd_multiplier(n)) >> 24);
}

/* ---- the kernel ---------------------------------------------------------------------------------- */
__global__ void __launch_bounds__(QS_RD_THREADS) qs_reduce_kernel(const QsReduceDesc *__restrict__ desc, int n) {
	int lo = 0, hi = n - 1;                                 /* the last picture whose first block is <= blockIdx.x */
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (desc[mid].blk <= blockIdx.x) lo = mid; else hi = mid - 1;
	}
	const QsReduceDesc d = desc[lo];
	const uint32_t len = (uint32_t)d.out_w * d.ch, per_row = (len + QS_RD_THREADS - 1) / QS_RD_THREADS, b = blockIdx.x - d.blk;
	const uint32_t y = b / per_row, j = (b - y * per_row) * QS_RD_THREADS + threadIdx.x;
	if (j < len) d.out[(size_t)y * len + j] = qs_rd_sample(d, y, j);
}

void qs_reduce_desc(const QsReducePlan &rd, int src_w, int ch, QsReduceDesc &d) {
	d.src_w = src_w; d.left = rd.left; d.top = rd.top; d.box_w = rd.box_w; d.box_h = rd.box_h;
	d.fx = rd.fx; d.fy = rd.fy; d.ch = ch; d.out_w = rd.out_w; d.out_h = rd.out_h; d.blk = 0;
}

uint32_t qs_reduce_number(QsReduceDesc *d, int n) {
	uint32_t b = 0;
	for (int i = 0; i < n; i++) {
		d[i].blk = b;
		b += (uint32_t)d[i].out_h * (((uint32_t)d[i].out_w * d[i].ch + QS_RD_THREADS - 1) / QS_RD_THREADS);
	}
	return b;
}

cudaError_t qs_launch_reduce(const QsReduceDesc *desc_dev, int n, uint32_t blocks, cudaStream_t st) {
	if (!n) return cudaSuccess;
	qs_reduce_kernel<<<blocks, QS_RD_THREADS, 0, st>>>(desc_dev, n);
	return cudaGetLastError();
}

/* ---- planning (host) ----------------------------------------------------------------------------- */
const char *qs_reduced_plan(int pic_w, int pic_h, const double box[4], int out_w, int out_h, int filter, double gap,
		QsReducePlan &rd, QsResizePlan &rp) {
	rd.fx = rd.fy = 1; rd.left = rd.top = 0; rd.box_w = rd.out_w = pic_w; rd.box_h = rd.out_h = pic_h;
	double b[4] = {box[0], box[1], box[2], box[3]};
	if (out_w < 1 || out_h < 1) return "output size below 1";
	if (gap > 0.0) {
		/* Image.resize: int(box_w / size_w / reducing_gap) or 1 per axis */
		const double fx = (b[2] - b[0]) / out_w / gap, fy = (b[3] - b[1]) / out_h / gap;
		if (fx >= 2.0 || fy >= 2.0) {
			rd.fx = fx < 2.0 ? 1 : (int)fx; rd.fy = fy < 2.0 ? 1 : (int)fy;
			if ((int64_t)rd.fx * rd.fy >= QS_REDUCE_MAX_CELL) return "the reduce's cell reaches 2^23 samples";
			/* _get_safe_box: the box widened by the filter's support less 0.5, in source samples */
			const double sup = qs_resize_support(filter) - 0.5;
			const double sx = sup * ((b[2] - b[0]) / out_w), sy = sup * ((b[3] - b[1]) / out_h);
			const int l = (int)(b[0] - sx), t = (int)(b[1] - sy);
			const int r = (int)ceil(b[2] + sx), bt = (int)ceil(b[3] + sy);
			rd.left = l < 0 ? 0 : l; rd.top = t < 0 ? 0 : t;
			rd.box_w = (r > pic_w ? pic_w : r) - rd.left; rd.box_h = (bt > pic_h ? pic_h : bt) - rd.top;
			rd.out_w = (rd.box_w + rd.fx - 1) / rd.fx; rd.out_h = (rd.box_h + rd.fy - 1) / rd.fy;
			b[0] = (b[0] - rd.left) / rd.fx; b[1] = (b[1] - rd.top) / rd.fy;
			b[2] = (b[2] - rd.left) / rd.fx; b[3] = (b[3] - rd.top) / rd.fy;
		}
	}
	if (rd.out_h > (int64_t)rd.out_w * 100 && out_h < rd.out_h) return "a picture more than 100 times taller than wide";
	const float fb[4] = {(float)b[0], (float)b[1], (float)b[2], (float)b[3]};
	return qs_resize_plan_box(rd.out_w, rd.out_h, fb, out_w, out_h, filter, rp);
}

/* round_aspect: of floor(v) and ceil(v), the first with the smaller error, at least 1 */
static int qs_round_aspect(double v, double aspect, int other, int x_axis) {
	const int f = (int)floor(v), c = (int)ceil(v);
	double kf, kc;
	if (x_axis) { kf = fabs(aspect - (double)f / other); kc = fabs(aspect - (double)c / other); }
	else { kf = f == 0 ? 0.0 : fabs(aspect - (double)other / f); kc = c == 0 ? 0.0 : fabs(aspect - (double)other / c); }
	const int n = kc < kf ? c : f;
	return n < 1 ? 1 : n;
}

void qs_thumbnail_geometry(int width, int height, int bound_w, int bound_h, double gap, int loaded, int *scale_denom,
		int *out_w, int *out_h) {
	*scale_denom = 1; *out_w = width; *out_h = height;
	if (bound_w >= width && bound_h >= height) return;     /* thumbnail returns before draft */
	const double aspect = (double)width / height;
	int x = bound_w, y = bound_h;
	if ((double)x / y >= aspect) x = qs_round_aspect(y * aspect, aspect, y, 1);
	else y = qs_round_aspect(x / aspect, aspect, x, 0);
	*out_w = x; *out_h = y;
	if (gap > 0.0 && !loaded) {
		/* JpegImageFile.draft(None, (int(w * gap), int(h * gap))) */
		const double gw = bound_w * gap, gh = bound_h * gap;
		const int sc_w = gw > width ? 0 : width / (int)gw, sc_h = gh > height ? 0 : height / (int)gh;
		const int sc = sc_w < sc_h ? sc_w : sc_h;
		*scale_denom = sc >= 8 ? 8 : sc >= 4 ? 4 : sc >= 2 ? 2 : 1;
	}
}

/* ---- the host models ----------------------------------------------------------------------------- */
static int model_fail(const char *who, const char *bad) {
	char m[200]; snprintf(m, sizeof(m), "%s: %s", who, bad);
	qs_set_host_error(m);
	return JPEGQS_ERR_ARG;
}

extern "C" int jpegqs_cuda_reduce_model(const uint8_t *src, int width, int height, int channels, int factor_x,
		int factor_y, const int32_t *box, uint8_t *out) {
	static const char who[] = "jpegqs_cuda_reduce_model";
	if (!src || !out) return model_fail(who, "NULL argument");
	if (width < 1 || height < 1) return model_fail(who, "picture size below 1");
	if (channels != 1 && channels != 3) return model_fail(who, "channels must be 1 or 3");
	if (factor_x < 1 || factor_y < 1) return model_fail(who, "factor below 1");
	if ((int64_t)factor_x * factor_y >= QS_REDUCE_MAX_CELL) return model_fail(who, "factor_x * factor_y reaches 2^23");
	QsReducePlan rd;
	const int32_t full[4] = {0, 0, width, height};
	const int32_t *b = box ? box : full;
	if (b[0] < 0 || b[1] < 0 || b[2] > width || b[3] > height || b[0] >= b[2] || b[1] >= b[3])
		return model_fail(who, "box outside the picture or empty");
	rd.fx = factor_x; rd.fy = factor_y; rd.left = b[0]; rd.top = b[1]; rd.box_w = b[2] - b[0]; rd.box_h = b[3] - b[1];
	rd.out_w = (rd.box_w + factor_x - 1) / factor_x; rd.out_h = (rd.box_h + factor_y - 1) / factor_y;
	QsReduceDesc d;
	qs_reduce_desc(rd, width, channels, d);
	d.src = src; d.out = out;
	const uint32_t len = (uint32_t)d.out_w * d.ch;
	for (uint32_t y = 0; y < (uint32_t)d.out_h; y++)
		for (uint32_t j = 0; j < len; j++) out[(size_t)y * len + j] = qs_rd_sample(d, y, j);
	return 0;
}

extern "C" int jpegqs_cuda_thumbnail_geometry(int width, int height, int bound_w, int bound_h, double reducing_gap,
		int loaded, int *scale_denom, int *out_w, int *out_h) {
	static const char who[] = "jpegqs_cuda_thumbnail_geometry";
	if (!scale_denom || !out_w || !out_h) return model_fail(who, "NULL argument");
	if (width < 1 || height < 1 || width > 65535 || height > 65535) return model_fail(who, "picture size outside 1..65535");
	if (bound_w < 1 || bound_h < 1 || bound_w > 65535 || bound_h > 65535) return model_fail(who, "bound outside 1..65535");
	if (!(reducing_gap == 0.0 || (isfinite(reducing_gap) && reducing_gap >= 1.0)))
		return model_fail(who, "reducing_gap must be 0 (None) or a finite value of at least 1.0");
	if (loaded != 0 && loaded != 1) return model_fail(who, "loaded must be 0 or 1");
	qs_thumbnail_geometry(width, height, bound_w, bound_h, reducing_gap, loaded, scale_denom, out_w, out_h);
	return 0;
}

extern "C" int jpegqs_cuda_resize_model_box(const uint8_t *src, int width, int height, int channels, int layout, int filter,
		const double *box, int out_w, int out_h, double reducing_gap, uint8_t *out) {
	static const char who[] = "jpegqs_cuda_resize_model_box";
	if (!src || !out) return model_fail(who, "NULL argument");
	if (width < 1 || height < 1) return model_fail(who, "picture size below 1");
	if (channels != 1 && channels != 3) return model_fail(who, "channels must be 1 or 3");
	if (layout != JPEGQS_RENDER_HWC && layout != JPEGQS_RENDER_CHW) return model_fail(who, "unknown layout");
	if (!qs_resize_filter_ok(filter)) return model_fail(who, "unknown filter (NEAREST is not a convolution filter)");
	if (!(reducing_gap == 0.0 || (isfinite(reducing_gap) && reducing_gap >= 1.0)))
		return model_fail(who, "reducing_gap must be 0 (None) or a finite value of at least 1.0");
	const double full[4] = {0.0, 0.0, (double)width, (double)height};
	const double *b = box ? box : full;
	if (!(b[0] >= 0.0 && b[1] >= 0.0 && b[2] <= width && b[3] <= height && b[0] < b[2] && b[1] < b[3]))
		return model_fail(who, "box outside the picture or empty");
	QsReducePlan rd; QsResizePlan rp;
	const char *bad = qs_reduced_plan(width, height, b, out_w, out_h, filter, reducing_gap, rd, rp);
	if (bad) return model_fail(who, bad);
	std::vector<uint8_t> red;
	const uint8_t *pic = src;
	if (rd.fx > 1 || rd.fy > 1) {
		red.resize((size_t)rd.out_w * rd.out_h * channels);
		QsReduceDesc d;
		qs_reduce_desc(rd, width, channels, d);
		d.src = src; d.out = red.data();
		const uint32_t len = (uint32_t)d.out_w * d.ch;
		for (uint32_t y = 0; y < (uint32_t)d.out_h; y++)
			for (uint32_t j = 0; j < len; j++) red[(size_t)y * len + j] = qs_rd_sample(d, y, j);
		pic = red.data();
	}
	qs_resize_run_model(rp, pic, rd.out_w, channels, layout == JPEGQS_RENDER_CHW, out);
	return 0;
}
