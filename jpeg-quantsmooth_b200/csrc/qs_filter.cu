/*
 * qs_filter.cu - blur and sharpen 8-bit pictures exactly as Pillow's ImageFilter.BoxBlur, GaussianBlur and
 * UnsharpMask do (libImaging/BoxBlur.c, UnsharpMask.c): the last stage of jpegqs_cuda_pixels_batch_filtered,
 * and jpegqs_cuda_image_filter_model, the same computation on one CPU thread.
 *
 * A box pass is integer arithmetic with one exact answer (include/jpegqs_cuda.h gives the rule).  The
 * window sum is an integer sum, so it is computed here in whatever order suits the pass, and no sample's
 * cost depends on the radius:
 *   - rows that fit QS_FILTER_ROW_MAX: one block per row holds the row in shared memory, and for each of
 *     the filter's row passes takes per-channel prefix sums of it and reads each window sum as a
 *     difference of two of them (qs_ft_prefix_sample).  One read and one write of the picture for all
 *     the row passes;
 *   - wider rows, and every column pass: one thread per line (a row's channel, or a column byte) slides
 *     the window down the line, adding the sample that enters and subtracting the one that leaves
 *     (qs_ft_line).  Column threads are consecutive bytes of a row, so every load and store is coalesced.
 * Pillow runs every row pass before the column passes and stores 8-bit samples between passes; so does
 * this.  UnsharpMask's comparison with its input is fused into the last column pass.
 *
 * Every launch covers every picture of a sub-batch; a block finds its picture by a binary search over the
 * pictures' first blocks, as the resize and reduce kernels do.  The gaussian box radius and the weights
 * are computed on the host, in float as Pillow types them; the device only adds and multiplies integers.
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "qs_filter.h"

extern "C" void qs_set_host_error(const char *msg);        /* qs_cuda.cu: jpegqs_cuda_last_error(NULL) */

#define QS_FT_THREADS 256
#define QS_FT_SMEM ((size_t)QS_FILTER_ROW_MAX * 5)          /* the widest row's prefix sums (uint32) and bytes */

/* ---- the per-sample arithmetic (device and host model) -------------------------------------------- */
__host__ __device__ static inline uint8_t qs_ft_round(uint32_t acc, uint32_t far, uint32_t ww, uint32_t fw) {
	return (uint8_t)((acc * ww + far * fw + (1u << 23)) >> 24);
}

/* UnsharpMask.c: in where |in - blur| <= threshold, else clip8(in + diff * percent / 100) */
__host__ __device__ static inline uint8_t qs_ft_unsharp(uint8_t in, uint8_t blur, int32_t percent, int32_t threshold) {
	const int32_t diff = (int32_t)in - (int32_t)blur;
	if ((diff < 0 ? -diff : diff) <= threshold) return in;
	const int32_t v = (int32_t)in + diff * percent / 100;
	return (uint8_t)(v <= 0 ? 0 : v >= 255 ? 255 : v);
}

/* sample x, channel c of a box pass over a row of n pixels of ch bytes, from its per-channel inclusive
 * prefix sums S[i * ch + c] = p[0] + ... + p[i] */
__host__ __device__ static inline uint8_t qs_ft_prefix_sample(const uint32_t *S, int32_t n, int32_t ch, int32_t x,
		int32_t c, int32_t r, uint32_t ww, uint32_t fw) {
	const int32_t last = n - 1, lo = x - r, hi = x + r, a = x - r - 1, b = x + r + 1;
	const uint32_t p0 = S[c], pl = S[last * ch + c] - (last ? S[(last - 1) * ch + c] : 0);
	uint32_t acc = S[(hi < last ? hi : last) * ch + c] - (lo > 0 ? S[(lo - 1) * ch + c] : 0);
	if (lo < 0) acc += (uint32_t)(-lo) * p0;
	if (hi > last) acc += (uint32_t)(hi - last) * pl;
	const uint32_t fa = a <= 0 ? p0 : S[a * ch + c] - S[(a - 1) * ch + c];
	const uint32_t fb = b >= last ? pl : S[b * ch + c] - S[(b - 1) * ch + c];
	return qs_ft_round(acc, fa + fb, ww, fw);
}

/* one box pass along a line of n samples src[i * ss] into dst[i * ds], the window slid one sample at a
 * time; orig != NULL: UnsharpMask's last pass, orig[i * ss] the filter's input */
__host__ __device__ static inline void qs_ft_line(const uint8_t *src, size_t ss, uint8_t *dst, size_t ds, const uint8_t *orig,
		int32_t n, const QsFilterDesc &d) {
	const int32_t last = n - 1, r = d.r;
	const int32_t m = r < last ? r : last;
	uint32_t acc = (uint32_t)src[0] * (uint32_t)(r + 1);
	for (int32_t k = 1; k <= m; k++) acc += src[(size_t)k * ss];
	if (r > last) acc += (uint32_t)(r - last) * src[(size_t)last * ss];
	uint32_t b = src[0];                                    /* p[c(x - r - 1)] */
	for (int32_t x = 0; x < n; x++) {
		const int32_t ia = x + r + 1, it = x - r;
		const uint32_t a = src[(size_t)(ia > last ? last : ia) * ss];
		const uint8_t v = qs_ft_round(acc, a + b, d.ww, d.fw);
		dst[(size_t)x * ds] = orig ? qs_ft_unsharp(orig[(size_t)x * ss], v, d.percent, d.threshold) : v;
		const uint32_t t = src[(size_t)(it < 0 ? 0 : it) * ss];
		acc += a - t;
		b = t;
	}
}

/* the last pass's store of sample (y, x, c): the caller's layout, UnsharpMask's comparison */
__host__ __device__ static inline void qs_ft_put(const QsFilterDesc &d, int32_t y, int32_t x, int32_t c, uint8_t v) {
	const size_t hwc = ((size_t)y * d.w + x) * d.ch + c;
	if (d.orig) v = qs_ft_unsharp(d.orig[hwc], v, d.percent, d.threshold);
	d.dst[d.chw ? ((size_t)c * d.h + y) * d.w + x : hwc] = v;
}

/* ---- the kernels --------------------------------------------------------------------------------- */
__device__ static inline int qs_ft_find(const QsFilterDesc *__restrict__ desc, int n) {
	int lo = 0, hi = n - 1;                                 /* the last picture whose first block is <= blockIdx.x */
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (desc[mid].blk <= blockIdx.x) lo = mid; else hi = mid - 1;
	}
	return lo;
}

/* the per-channel inclusive prefix sums of row (n pixels of ch bytes) into S: each thread sums a segment
 * of consecutive pixels, the segments' totals are scanned across the block, and each thread writes its
 * segment's sums.  Ends with a barrier. */
__device__ static void qs_ft_scan(const uint8_t *row, uint32_t *S, int32_t n, int32_t ch) {
	__shared__ uint32_t s_warp[QS_FT_THREADS / 32][3];
	const int32_t seg = (n + QS_FT_THREADS - 1) / QS_FT_THREADS, x0 = threadIdx.x * seg;
	const int32_t x1 = x0 + seg < n ? x0 + seg : n;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t tot[3] = {0, 0, 0};
	for (int32_t x = x0; x < x1; x++)
		for (int32_t c = 0; c < ch; c++) tot[c] += row[x * ch + c];
	uint32_t inc[3];
	for (int c = 0; c < 3; c++) {
		inc[c] = tot[c];
		for (int s = 1; s < 32; s <<= 1) {
			const uint32_t o = __shfl_up_sync(0xffffffffu, inc[c], s);
			if (lane >= s) inc[c] += o;
		}
		if (lane == 31) s_warp[warp][c] = inc[c];
	}
	__syncthreads();
	for (int c = 0; c < 3; c++) {
		uint32_t run = inc[c] - tot[c];
		for (int w = 0; w < warp; w++) run += s_warp[w][c];
		tot[c] = run;
	}
	for (int32_t x = x0; x < x1; x++)
		for (int32_t c = 0; c < ch; c++) { tot[c] += row[x * ch + c]; S[x * ch + c] = tot[c]; }
	__syncthreads();
}

/* rows that fit QS_FILTER_ROW_MAX: block b is one row; every row pass in shared memory (5 bytes per byte of
 * the launch's widest row: the prefix sums, then the row) */
__global__ void __launch_bounds__(QS_FT_THREADS) qs_filter_rows_kernel(const QsFilterDesc *__restrict__ desc, int n) {
	extern __shared__ uint32_t s_sum[];
	const QsFilterDesc d = desc[qs_ft_find(desc, n)];
	const int32_t y = blockIdx.x - d.blk, len = d.w * d.ch;
	uint8_t *row = (uint8_t*)(s_sum + len);
	const uint8_t *src = d.src + (size_t)y * len;
	for (int32_t j = threadIdx.x; j < len; j += QS_FT_THREADS) row[j] = src[j];
	for (int32_t pass = 0; pass < d.npass; pass++) {
		__syncthreads();
		qs_ft_scan(row, s_sum, d.w, d.ch);
		const bool last = pass == d.npass - 1;
		for (int32_t j = threadIdx.x; j < len; j += QS_FT_THREADS) {
			const int32_t x = j / d.ch, c = j - x * d.ch;
			const uint8_t v = qs_ft_prefix_sample(s_sum, d.w, d.ch, x, c, d.r, d.ww, d.fw);
			if (last) qs_ft_put(d, y, x, c, v); else row[j] = v;
		}
	}
}

/* one row pass over rows wider than QS_FILTER_ROW_MAX: thread t is one channel of one row */
__global__ void __launch_bounds__(QS_FT_THREADS) qs_filter_wide_kernel(const QsFilterDesc *__restrict__ desc, int n) {
	const QsFilterDesc d = desc[qs_ft_find(desc, n)];
	const uint32_t line = (blockIdx.x - d.blk) * QS_FT_THREADS + threadIdx.x;
	if (line >= (uint32_t)d.h * d.ch) return;
	const int32_t y = line / d.ch, c = line - y * d.ch;
	const size_t off = (size_t)y * d.w * d.ch + c;
	if (d.chw) qs_ft_line(d.src + off, d.ch, d.dst + ((size_t)c * d.h + y) * d.w, 1, d.orig ? d.orig + off : NULL, d.w, d);
	else qs_ft_line(d.src + off, d.ch, d.dst + off, d.ch, d.orig ? d.orig + off : NULL, d.w, d);
}

/* one column pass: thread t is one byte column (x, c), consecutive threads consecutive bytes of a row */
__global__ void __launch_bounds__(QS_FT_THREADS) qs_filter_cols_kernel(const QsFilterDesc *__restrict__ desc, int n) {
	const QsFilterDesc d = desc[qs_ft_find(desc, n)];
	const uint32_t j = (blockIdx.x - d.blk) * QS_FT_THREADS + threadIdx.x, len = (uint32_t)d.w * d.ch;
	if (j >= len) return;
	if (d.chw) {
		const int32_t x = j / d.ch, c = j - x * d.ch;
		qs_ft_line(d.src + j, len, d.dst + (size_t)c * d.h * d.w + x, d.w, d.orig ? d.orig + j : NULL, d.h, d);
	} else {
		qs_ft_line(d.src + j, len, d.dst + j, len, d.orig ? d.orig + j : NULL, d.h, d);
	}
}

cudaError_t qs_filter_enqueue(const std::vector<QsFilterLaunch> &launches, const QsFilterDesc *desc_dev, cudaStream_t st) {
	for (const QsFilterLaunch &l : launches) {
		if (!l.count) continue;
		const QsFilterDesc *d = desc_dev + l.first;
		if (l.kind == QS_FILTER_ROWS) {
			cudaError_t e = cudaFuncSetAttribute(qs_filter_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)QS_FT_SMEM);
			if (e != cudaSuccess) return e;
			qs_filter_rows_kernel<<<l.blocks, QS_FT_THREADS, l.smem, st>>>(d, l.count);
		} else if (l.kind == QS_FILTER_WIDE) {
			qs_filter_wide_kernel<<<l.blocks, QS_FT_THREADS, 0, st>>>(d, l.count);
		} else {
			qs_filter_cols_kernel<<<l.blocks, QS_FT_THREADS, 0, st>>>(d, l.count);
		}
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess) return e;
	}
	return cudaSuccess;
}

/* ---- planning (host) ----------------------------------------------------------------------------- */
/* BoxBlur.c's _gaussian_blur_radius(s, 3), typed as Pillow types it */
static float qs_ft_gauss_box(float radius) {
	const float sigma2 = radius * radius / 3;
	const float L = (float)sqrt(12.0 * sigma2 + 1.0);
	const float l = (float)floor((L - 1.0) / 2.0);
	float a = (2 * l + 1) * (l * (l + 1) - 3 * sigma2);
	a /= 6 * (sigma2 - (l + 1) * (l + 1));
	return l + a;
}

const char *qs_filter_check(const jpegqs_cuda_image_filter &f) {
	if (f.kind != JPEGQS_FILTER_BOX_BLUR && f.kind != JPEGQS_FILTER_GAUSSIAN_BLUR && f.kind != JPEGQS_FILTER_UNSHARP_MASK)
		return "unknown filter kind (expected BOX_BLUR 1, GAUSSIAN_BLUR 2 or UNSHARP_MASK 3)";
	if (!(fabsf(f.radius_x) <= JPEGQS_FILTER_MAX_RADIUS && fabsf(f.radius_y) <= JPEGQS_FILTER_MAX_RADIUS))
		return "radius not finite or above 65535";
	if (f.kind == JPEGQS_FILTER_BOX_BLUR && (f.radius_x < 0 || f.radius_y < 0)) return "radius must be >= 0";
	if (f.kind == JPEGQS_FILTER_UNSHARP_MASK) {
		if (f.radius_x != f.radius_y) return "UNSHARP_MASK takes one radius (radius_x = radius_y)";
		if (f.percent < -JPEGQS_FILTER_MAX_PERCENT || f.percent > JPEGQS_FILTER_MAX_PERCENT)
			return "percent outside -8421504..8421504 (|diff * percent| would reach 2^31)";
	}
	return NULL;
}

/* one axis of one filter: its pass count (0 skips the axis: radius 0, whose pass is the identity), radius
 * and weights */
struct QsFtAxis { int passes; int32_t r; uint32_t ww, fw; };
static QsFtAxis qs_ft_axis(float R, int passes) {
	QsFtAxis a;
	a.passes = R == 0.0f ? 0 : passes; a.r = (int32_t)R;
	a.ww = (uint32_t)(16777216.0f / (R * 2.0f + 1.0f));
	a.fw = (16777216u - (uint32_t)(a.r * 2 + 1) * a.ww) / 2;
	return a;
}

void qs_filter_plan(const jpegqs_cuda_image_filter *f, int nf, const QsFilterPic *pics, int n,
		std::vector<QsFilterDesc> &desc, std::vector<QsFilterLaunch> &launches) {
	desc.clear(); launches.clear();
	std::vector<uint8_t*> cur_in((size_t)n);
	for (int i = 0; i < n; i++) cur_in[i] = pics[i].in;
	for (int k = 0; k < nf; k++) {
		const bool last_filter = k == nf - 1, unsharp = f[k].kind == JPEGQS_FILTER_UNSHARP_MASK;
		QsFtAxis ax[2];
		if (f[k].kind == JPEGQS_FILTER_BOX_BLUR) {
			ax[0] = qs_ft_axis(f[k].radius_x, 1); ax[1] = qs_ft_axis(f[k].radius_y, 1);
		} else {
			ax[0] = qs_ft_axis(qs_ft_gauss_box(f[k].radius_x), 3); ax[1] = qs_ft_axis(qs_ft_gauss_box(f[k].radius_y), 3);
		}
		/* the launches of this filter, in order: fused rows, wide rows 1..3, columns 1..3 */
		std::vector<QsFilterDesc> bucket[QS_FILTER_MAX_STEPS];
		for (int i = 0; i < n; i++) {
			const QsFilterPic &p = pics[i];
			const bool fused = (size_t)p.w * p.ch <= QS_FILTER_ROW_MAX;
			struct Step { int bucket; QsFtAxis a; int npass; };
			std::vector<Step> steps;
			if (ax[0].passes && fused) steps.push_back({0, ax[0], ax[0].passes});
			else for (int q = 0; q < ax[0].passes; q++) steps.push_back({1 + q, ax[0], 1});
			for (int q = 0; q < ax[1].passes; q++) steps.push_back({4 + q, ax[1], 1});
			if (steps.empty()) {
				/* nothing to blur: the input as it is (UnsharpMask of an unblurred picture is its input) */
				if (!last_filter) continue;
				steps.push_back({4, qs_ft_axis(0.0f, 1), 1});
			}
			/* ping-pong between the two buffers that are not the filter's input; the last pass writes the
			 * destination, or the next filter's input (never the line's own source: a line pass reads
			 * samples behind the one it writes) */
			uint8_t *in = cur_in[i], *o0 = p.in == in ? p.a : p.in, *o1 = p.b == in ? p.a : p.b;
			const uint8_t *cur = in;
			for (size_t s = 0; s < steps.size(); s++) {
				const bool last = s + 1 == steps.size();
				uint8_t *dst = last ? (last_filter ? p.out : (cur != in ? in : o0)) : (cur == o0 ? o1 : o0);
				QsFilterDesc d;
				memset(&d, 0, sizeof(d));
				d.src = cur; d.dst = dst; d.orig = last && unsharp ? in : NULL;
				d.w = p.w; d.h = p.h; d.ch = p.ch; d.chw = last && last_filter ? p.chw : 0;
				d.r = steps[s].a.r; d.npass = steps[s].npass; d.ww = steps[s].a.ww; d.fw = steps[s].a.fw;
				d.percent = f[k].percent; d.threshold = f[k].threshold;
				bucket[steps[s].bucket].push_back(d);
				cur = dst;
			}
			cur_in[i] = (uint8_t*)cur;
		}
		for (int b = 0; b < QS_FILTER_MAX_STEPS; b++) {
			if (bucket[b].empty()) continue;
			QsFilterLaunch l;
			l.kind = b == 0 ? QS_FILTER_ROWS : b < 4 ? QS_FILTER_WIDE : QS_FILTER_COLS;
			l.first = (int)desc.size(); l.count = (int)bucket[b].size(); l.smem = 0;
			uint32_t blk = 0;
			for (QsFilterDesc &d : bucket[b]) {
				d.blk = blk;
				const uint32_t lines = l.kind == QS_FILTER_ROWS ? (uint32_t)d.h :
						(((uint32_t)(l.kind == QS_FILTER_WIDE ? d.h : d.w) * d.ch + QS_FT_THREADS - 1) / QS_FT_THREADS);
				blk += lines;
				if (b == 0 && (size_t)d.w * d.ch * 5 > l.smem) l.smem = ((size_t)d.w * d.ch * 5 + 15) & ~(size_t)15;
				desc.push_back(d);
			}
			l.blocks = blk;
			launches.push_back(l);
		}
	}
}

/* ---- the host model ------------------------------------------------------------------------------ */
static int model_fail(const char *bad) {
	char m[200]; snprintf(m, sizeof(m), "jpegqs_cuda_image_filter_model: %s", bad);
	qs_set_host_error(m);
	return JPEGQS_ERR_ARG;
}

extern "C" int jpegqs_cuda_image_filter_model(const uint8_t *src, int width, int height, int channels,
		const jpegqs_cuda_image_filter *filters, int nfilters, uint8_t *out) {
	if (!src || !out || (nfilters && !filters)) return model_fail("NULL argument");
	if (width < 1 || height < 1) return model_fail("picture size below 1");
	if (channels != 1 && channels != 3) return model_fail("channels must be 1 or 3");
	if (nfilters < 0 || nfilters > 64) return model_fail("nfilters outside 0..64");
	for (int k = 0; k < nfilters; k++) {
		const char *bad = qs_filter_check(filters[k]);
		if (bad) { char m[160]; snprintf(m, sizeof(m), "filter %d: %s", k, bad); return model_fail(m); }
	}
	const size_t bytes = (size_t)width * height * channels;
	if (!nfilters) { memcpy(out, src, bytes); return 0; }
	std::vector<uint8_t> buf(3 * bytes);
	memcpy(buf.data(), src, bytes);
	QsFilterPic pic = {buf.data(), buf.data() + bytes, buf.data() + 2 * bytes, out, width, height, channels, 0};
	std::vector<QsFilterDesc> desc;
	std::vector<QsFilterLaunch> launches;
	qs_filter_plan(filters, nfilters, &pic, 1, desc, launches);
	std::vector<uint32_t> S((size_t)width * channels);
	std::vector<uint8_t> row((size_t)width * channels);
	for (const QsFilterLaunch &l : launches) {
		const QsFilterDesc &d = desc[l.first];
		const size_t len = (size_t)d.w * d.ch;
		if (l.kind == QS_FILTER_ROWS) {
			for (int32_t y = 0; y < d.h; y++) {
				memcpy(row.data(), d.src + y * len, len);
				for (int32_t pass = 0; pass < d.npass; pass++) {
					for (int32_t c = 0; c < d.ch; c++) {
						uint32_t s = 0;
						for (int32_t x = 0; x < d.w; x++) { s += row[(size_t)x * d.ch + c]; S[(size_t)x * d.ch + c] = s; }
					}
					std::vector<uint8_t> next(len);
					for (int32_t x = 0; x < d.w; x++)
						for (int32_t c = 0; c < d.ch; c++)
							next[(size_t)x * d.ch + c] = qs_ft_prefix_sample(S.data(), d.w, d.ch, x, c, d.r, d.ww, d.fw);
					if (pass + 1 < d.npass) row = next;
					else for (int32_t x = 0; x < d.w; x++) for (int32_t c = 0; c < d.ch; c++) qs_ft_put(d, y, x, c, next[(size_t)x * d.ch + c]);
				}
			}
		} else if (l.kind == QS_FILTER_WIDE) {
			for (int32_t y = 0; y < d.h; y++)
				for (int32_t c = 0; c < d.ch; c++) {
					const size_t off = (size_t)y * len + c;
					qs_ft_line(d.src + off, d.ch, d.dst + off, d.ch, d.orig ? d.orig + off : NULL, d.w, d);
				}
		} else {
			for (size_t j = 0; j < len; j++) qs_ft_line(d.src + j, len, d.dst + j, len, d.orig ? d.orig + j : NULL, d.h, d);
		}
	}
	return 0;
}
