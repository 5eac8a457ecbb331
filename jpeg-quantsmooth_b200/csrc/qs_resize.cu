/*
 * qs_resize.cu - crop and resize 8-bit pictures exactly as Pillow's Image.resize does with its
 * convolution filters (libImaging/Resample.c): the last stage of jpegqs_cuda_pixels_batch_resized,
 * and jpegqs_cuda_resize_model, the same computation on one CPU thread.
 *
 * Pillow computes each axis's weights in double (precompute_coeffs), rounds them to int32 with 22
 * fractional bits (normalize_coeffs_8bpc) and runs a horizontal pass, then a vertical one, in integer
 * arithmetic; each pass rounds and clamps its result to 8 bits.  The weights are built here on the host
 * with the same expressions, so sin and cos are glibc's, as Pillow's are; the device only multiplies
 * and adds integers, so its bytes are fully determined.  Pillow skips a pass over an axis whose size
 * does not change; that pass is an exact identity for every filter (the weight at distance 0 rounds to
 * 1 << 22, the others to 0), so both passes always run here.
 *
 * Each pass is one launch over every picture of a sub-batch.  A block takes up to QS_RS_THREADS
 * consecutive bytes of one output row, one byte per thread; a block finds its picture by a binary
 * search over the pictures' first blocks.
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <vector>
#include "qs_resize.h"

extern "C" void qs_set_host_error(const char *msg);        /* qs_cuda.cu: jpegqs_cuda_last_error(NULL) */

#define QS_RS_THREADS 256
#define QS_RS_BITS 22                                       /* Resample.c PRECISION_BITS */

/* ---- the weights (host) ------------------------------------------------------------------------ */
static double qs_rs_sinc(double x) {
	if (x == 0.0) return 1.0;
	x = x * M_PI;
	return sin(x) / x;
}

/* Resample.c's filters, expression for expression */
static double qs_rs_filter(int filter, double x) {
	switch (filter) {
	case JPEGQS_RESIZE_BOX:
		return x > -0.5 && x <= 0.5 ? 1.0 : 0.0;
	case JPEGQS_RESIZE_BILINEAR:
		if (x < 0.0) x = -x;
		return x < 1.0 ? 1.0 - x : 0.0;
	case JPEGQS_RESIZE_HAMMING:
		if (x < 0.0) x = -x;
		if (x == 0.0) return 1.0;
		if (x >= 1.0) return 0.0;
		x = x * M_PI;
		return sin(x) / x * (0.54f + 0.46f * cos(x));
	case JPEGQS_RESIZE_BICUBIC: {
		const double a = -0.5;
		if (x < 0.0) x = -x;
		if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
		if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
		return 0.0;
	}
	default:                                                /* LANCZOS: sinc truncated at 3 lobes */
		return -3.0 <= x && x < 3.0 ? qs_rs_sinc(x) * qs_rs_sinc(x / 3) : 0.0;
	}
}

double qs_resize_support(int filter) {
	return filter == JPEGQS_RESIZE_BOX ? 0.5 : filter == JPEGQS_RESIZE_BICUBIC ? 2.0 : filter == JPEGQS_RESIZE_LANCZOS ? 3.0 : 1.0;
}

int qs_resize_filter_ok(int filter) { return filter >= JPEGQS_RESIZE_LANCZOS && filter <= JPEGQS_RESIZE_HAMMING; }

/* precompute_coeffs + normalize_coeffs_8bpc for out_size samples centred at in0 + (xx + 0.5) * scale of
 * in_size: the bounds (first sample, count) and the rounded weights (row stride ksize, unused entries 0);
 * returns ksize */
static int qs_rs_axis_at(int in_size, double in0, double scale, int out_size, int filter, std::vector<int32_t> &bounds,
		std::vector<int32_t> &kk) {
	const double filterscale = scale < 1.0 ? 1.0 : scale;
	const double support = qs_resize_support(filter) * filterscale;
	const int ksize = (int)ceil(support) * 2 + 1;
	std::vector<double> w((size_t)ksize);
	bounds.assign((size_t)out_size * 2, 0);
	kk.assign((size_t)out_size * ksize, 0);
	for (int xx = 0; xx < out_size; xx++) {
		const double center = in0 + (xx + 0.5) * scale, ss = 1.0 / filterscale;
		double ww = 0.0;
		int xmin = (int)(center - support + 0.5);
		if (xmin < 0) xmin = 0;
		int xmax = (int)(center + support + 0.5);
		if (xmax > in_size) xmax = in_size;
		xmax -= xmin;
		for (int x = 0; x < xmax; x++) { w[x] = qs_rs_filter(filter, (x + xmin - center + 0.5) * ss); ww += w[x]; }
		for (int x = 0; x < xmax; x++) {
			if (ww != 0.0) w[x] /= ww;
			kk[(size_t)xx * ksize + x] = w[x] < 0 ? (int32_t)(-0.5 + w[x] * (1 << QS_RS_BITS)) : (int32_t)(0.5 + w[x] * (1 << QS_RS_BITS));
		}
		bounds[2 * xx] = xmin; bounds[2 * xx + 1] = xmax;
	}
	return ksize;
}

/* the whole of in_size -> out_size */
static int qs_rs_axis(int in_size, int out_size, int filter, std::vector<int32_t> &bounds, std::vector<int32_t> &kk) {
	return qs_rs_axis_at(in_size, 0.0, (double)in_size / out_size, out_size, filter, bounds, kk);
}

/* the plan from both axes' tables: the rows the vertical pass reads (bounds are monotonic) are the only
 * ones the horizontal pass makes */
static void qs_rs_finish(int l, int t, int out_w, int out_h, std::vector<int32_t> &hb, std::vector<int32_t> &hk,
		std::vector<int32_t> &vb, std::vector<int32_t> &vk, QsResizePlan &rp) {
	const int first = vb[0], last = vb[2 * (out_h - 1)] + vb[2 * (out_h - 1) + 1];
	for (int y = 0; y < out_h; y++) vb[2 * y] -= first;
	rp.left = l; rp.top = t + first; rp.out_w = out_w; rp.out_h = out_h; rp.mid_h = last - first;
	rp.tab.clear();
	rp.tab.reserve(hb.size() + hk.size() + vb.size() + vk.size());
	for (const std::vector<int32_t> *v : {&hb, &hk, &vb, &vk}) rp.tab.insert(rp.tab.end(), v->begin(), v->end());
}

const char *qs_resize_plan(int pic_w, int pic_h, const jpegqs_cuda_resize_box &box, int filter, QsResizePlan &rp) {
	if (box.width < 1 || box.width > 65535 || box.height < 1 || box.height > 65535) return "output size outside 1..65535";
	int l = box.left, t = box.top, r = box.right, b = box.bottom;
	if (!l && !t && !r && !b) { r = pic_w; b = pic_h; }
	if (l < 0 || t < 0 || r > pic_w || b > pic_h) return "crop outside the picture";
	if (l >= r || t >= b) return "empty crop";
	std::vector<int32_t> hb, hk, vb, vk;
	rp.ksh = qs_rs_axis(r - l, box.width, filter, hb, hk);
	rp.ksv = qs_rs_axis(b - t, box.height, filter, vb, vk);
	qs_rs_finish(l, t, box.width, box.height, hb, hk, vb, vk, rp);
	return NULL;
}

/* Pillow's C layer takes the box as float: scale = (double)(float)(in1 - in0) / out, and each centre is
 * in0 + (xx + 0.5) * scale in double, over the whole picture (samples outside the box are read) */
const char *qs_resize_plan_box(int pic_w, int pic_h, const float box[4], int out_w, int out_h, int filter, QsResizePlan &rp) {
	if (out_w < 1 || out_w > 65535 || out_h < 1 || out_h > 65535) return "output size outside 1..65535";
	if (!(box[0] >= 0.0f && box[1] >= 0.0f && box[2] <= (float)pic_w && box[3] <= (float)pic_h)) return "box outside the picture";
	if (!(box[2] > box[0] && box[3] > box[1])) return "empty box";
	std::vector<int32_t> hb, hk, vb, vk;
	rp.ksh = qs_rs_axis_at(pic_w, box[0], (double)(float)(box[2] - box[0]) / out_w, out_w, filter, hb, hk);
	rp.ksv = qs_rs_axis_at(pic_h, box[1], (double)(float)(box[3] - box[1]) / out_h, out_h, filter, vb, vk);
	qs_rs_finish(0, 0, out_w, out_h, hb, hk, vb, vk, rp);
	return NULL;
}

void qs_resize_desc(const QsResizePlan &rp, int src_w, int ch, int chw, QsResizeDesc &d) {
	d.src_w = src_w; d.left = rp.left; d.top = rp.top; d.out_w = rp.out_w; d.out_h = rp.out_h; d.mid_h = rp.mid_h;
	d.ksh = rp.ksh; d.ksv = rp.ksv; d.ch = ch; d.chw = ch == 3 && chw;
	d.hblk = d.vblk = 0;
}

/* ---- the per-pixel arithmetic (device and host model) --------------------------------------------
 * A row of each pass: the horizontal pass has mid_h rows of out_w * ch bytes; the vertical pass has
 * out_h rows of out_w * ch bytes (HWC), or ch * out_h rows of out_w bytes (CHW, row c * out_h + yy). */
__host__ __device__ static inline uint8_t qs_rs_clip8(int32_t ss) {
	ss >>= QS_RS_BITS;
	return (uint8_t)(ss < 0 ? 0 : ss > 255 ? 255 : ss);
}

/* 1 << 21, plus n taps of src (stride bytes apart) times k, clipped: Resample.c's inner loop */
__host__ __device__ static inline uint8_t qs_rs_dot(const uint8_t *src, size_t stride, const int32_t *k, int n) {
	int32_t ss = 1 << (QS_RS_BITS - 1);
	for (int i = 0; i < n; i++) ss += (int32_t)src[(size_t)i * stride] * k[i];
	return qs_rs_clip8(ss);
}

__host__ __device__ static inline uint32_t qs_rs_hlen(const QsResizeDesc &d) { return (uint32_t)d.out_w * d.ch; }
__host__ __device__ static inline uint32_t qs_rs_vlen(const QsResizeDesc &d) { return d.chw ? (uint32_t)d.out_w : (uint32_t)d.out_w * d.ch; }
__host__ __device__ static inline uint32_t qs_rs_vrows(const QsResizeDesc &d) { return d.chw ? (uint32_t)d.out_h * d.ch : (uint32_t)d.out_h; }

/* byte j of intermediate row y */
__host__ __device__ static inline uint8_t qs_rs_h(const QsResizeDesc &d, uint32_t y, uint32_t j) {
	const uint32_t xx = j / d.ch, c = j - xx * d.ch;
	const int32_t *b = d.tab + 2 * xx;
	const int32_t *k = d.tab + 2 * (size_t)d.out_w + (size_t)xx * d.ksh;
	const uint8_t *s = d.src + ((size_t)(d.top + y) * d.src_w + d.left + b[0]) * d.ch + c;
	return qs_rs_dot(s, d.ch, k, b[1]);
}

/* byte j of output row r */
__host__ __device__ static inline uint8_t qs_rs_v(const QsResizeDesc &d, uint32_t r, uint32_t j) {
	uint32_t yy, xx, c;
	if (d.chw) { c = r / d.out_h; yy = r - c * d.out_h; xx = j; }
	else { yy = r; xx = j / d.ch; c = j - xx * d.ch; }
	const int32_t *vb = d.tab + 2 * (size_t)d.out_w + (size_t)d.out_w * d.ksh;
	const int32_t *k = vb + 2 * (size_t)d.out_h + (size_t)yy * d.ksv;
	const size_t stride = (size_t)d.out_w * d.ch;
	const uint8_t *s = d.mid + (size_t)vb[2 * yy] * stride + (size_t)xx * d.ch + c;
	return qs_rs_dot(s, stride, k, vb[2 * yy + 1]);
}

/* ---- the kernels --------------------------------------------------------------------------------- */
/* the last picture whose first block is <= blk (every picture has at least one block) */
__device__ static inline int qs_rs_find(const QsResizeDesc *__restrict__ desc, int n, uint32_t blk, bool vert) {
	int lo = 0, hi = n - 1;
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if ((vert ? desc[mid].vblk : desc[mid].hblk) <= blk) lo = mid; else hi = mid - 1;
	}
	return lo;
}

__global__ void __launch_bounds__(QS_RS_THREADS) qs_resize_h_kernel(const QsResizeDesc *__restrict__ desc, int n) {
	const QsResizeDesc d = desc[qs_rs_find(desc, n, blockIdx.x, false)];
	const uint32_t len = qs_rs_hlen(d), per_row = (len + QS_RS_THREADS - 1) / QS_RS_THREADS, b = blockIdx.x - d.hblk;
	const uint32_t y = b / per_row, j = (b - y * per_row) * QS_RS_THREADS + threadIdx.x;
	if (j < len) d.mid[(size_t)y * len + j] = qs_rs_h(d, y, j);
}

__global__ void __launch_bounds__(QS_RS_THREADS) qs_resize_v_kernel(const QsResizeDesc *__restrict__ desc, int n) {
	const QsResizeDesc d = desc[qs_rs_find(desc, n, blockIdx.x, true)];
	const uint32_t len = qs_rs_vlen(d), per_row = (len + QS_RS_THREADS - 1) / QS_RS_THREADS, b = blockIdx.x - d.vblk;
	const uint32_t r = b / per_row, j = (b - r * per_row) * QS_RS_THREADS + threadIdx.x;
	if (j < len) d.out[(size_t)r * len + j] = qs_rs_v(d, r, j);
}

void qs_resize_number(QsResizeDesc *d, int n, uint32_t *hblocks, uint32_t *vblocks) {
	uint32_t h = 0, v = 0;
	for (int i = 0; i < n; i++) {
		d[i].hblk = h; d[i].vblk = v;
		h += (uint32_t)d[i].mid_h * ((qs_rs_hlen(d[i]) + QS_RS_THREADS - 1) / QS_RS_THREADS);
		v += qs_rs_vrows(d[i]) * ((qs_rs_vlen(d[i]) + QS_RS_THREADS - 1) / QS_RS_THREADS);
	}
	*hblocks = h; *vblocks = v;
}

cudaError_t qs_launch_resize(const QsResizeDesc *desc_dev, int n, uint32_t hblocks, uint32_t vblocks, cudaStream_t st) {
	if (!n) return cudaSuccess;
	qs_resize_h_kernel<<<hblocks, QS_RS_THREADS, 0, st>>>(desc_dev, n);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return e;
	qs_resize_v_kernel<<<vblocks, QS_RS_THREADS, 0, st>>>(desc_dev, n);
	return cudaGetLastError();
}

/* ---- the host model ------------------------------------------------------------------------------ */
extern "C" int jpegqs_cuda_resize_model(const uint8_t *src, int width, int height, int channels, int layout, int filter,
		const jpegqs_cuda_resize_box *box, uint8_t *out) {
	QsResizePlan rp;
	const char *bad = !src || !box || !out ? "NULL argument" : width < 1 || height < 1 ? "picture size below 1" :
			channels != 1 && channels != 3 ? "channels must be 1 or 3" :
			layout != JPEGQS_RENDER_HWC && layout != JPEGQS_RENDER_CHW ? "unknown layout" :
			!qs_resize_filter_ok(filter) ? "unknown filter (NEAREST is not a convolution filter)" : NULL;
	if (!bad) bad = qs_resize_plan(width, height, *box, filter, rp);
	if (bad) {
		char m[160]; snprintf(m, sizeof(m), "jpegqs_cuda_resize_model: %s", bad);
		qs_set_host_error(m);
		return JPEGQS_ERR_ARG;
	}
	qs_resize_run_model(rp, src, width, channels, layout == JPEGQS_RENDER_CHW, out);
	return 0;
}

void qs_resize_run_model(const QsResizePlan &rp, const uint8_t *src, int src_w, int ch, int chw, uint8_t *out) {
	QsResizeDesc d;
	qs_resize_desc(rp, src_w, ch, chw, d);
	std::vector<uint8_t> mid((size_t)d.mid_h * qs_rs_hlen(d));
	d.src = src; d.mid = mid.data(); d.out = out; d.tab = rp.tab.data();
	for (uint32_t y = 0; y < (uint32_t)d.mid_h; y++)
		for (uint32_t j = 0; j < qs_rs_hlen(d); j++) mid[(size_t)y * qs_rs_hlen(d) + j] = qs_rs_h(d, y, j);
	for (uint32_t r = 0; r < qs_rs_vrows(d); r++)
		for (uint32_t j = 0; j < qs_rs_vlen(d); j++) out[(size_t)r * qs_rs_vlen(d) + j] = qs_rs_v(d, r, j);
}
