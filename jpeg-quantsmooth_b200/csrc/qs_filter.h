/* qs_filter.h - the filter stage of jpegqs_cuda_pixels_batch_filtered (qs_filter.cu): Pillow's
 * ImageFilter.BoxBlur, GaussianBlur and UnsharpMask (libImaging/BoxBlur.c, UnsharpMask.c) of 8-bit HWC
 * pictures, byte for byte. */
#ifndef QS_FILTER_H
#define QS_FILTER_H

#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include "../../include/jpegqs_cuda.h"

/* The largest row (width x channels bytes) whose passes the row kernel fuses in shared memory: the row
 * and its uint32 prefix sums, 80 KB, two blocks per SM.  Wider rows take one launch per pass. */
#define QS_FILTER_ROW_MAX 16384

/* One pass (or, in the row kernel, npass fused passes) of one picture on the device, or in the host model
 * with host pointers.  src and every intermediate are HWC (w x h x ch); the filter's last pass writes dst
 * in the caller's layout (chw: ch planes) and, for UnsharpMask, compares with orig (the filter's input,
 * HWC).  r, ww, fw: BoxBlur.c's window radius (int)R and its two weights. */
struct QsFilterDesc {
	const uint8_t *src;
	uint8_t *dst;
	const uint8_t *orig;         /* UnsharpMask's last pass: its input; else NULL */
	int32_t w, h, ch, chw;
	int32_t r, npass;
	uint32_t ww, fw;
	int32_t percent, threshold;
	uint32_t blk;                /* the picture's first block in the launch */
	int32_t pad;
};

/* One launch of the chain: kind, its descriptors desc[first .. first + count), its grid and (rows) its
 * dynamic shared memory. */
enum { QS_FILTER_ROWS = 0, QS_FILTER_WIDE = 1, QS_FILTER_COLS = 2 };
struct QsFilterLaunch {
	int kind, first, count;
	uint32_t blocks;
	size_t smem;
};

/* One picture of the chain: its input `in` (HWC, overwritten by the chain), two scratch pictures of the
 * same size, and the destination of the last filter's last pass in layout chw. */
struct QsFilterPic {
	uint8_t *in, *a, *b, *out;
	int32_t w, h, ch, chw;
};

/* NULL, or why the filter is refused (kind, radii, percent) */
const char *qs_filter_check(const jpegqs_cuda_image_filter &f);
/* the descriptors and launches of filters[0..nf) applied in order to every picture */
void qs_filter_plan(const jpegqs_cuda_image_filter *f, int nf, const QsFilterPic *pics, int n,
		std::vector<QsFilterDesc> &desc, std::vector<QsFilterLaunch> &launches);
/* the most launches and descriptors per picture one filter makes (sizing of the descriptor upload) */
#define QS_FILTER_MAX_STEPS 7
/* the launches over descriptors already in device memory (desc_dev: the plan's desc, uploaded) */
cudaError_t qs_filter_enqueue(const std::vector<QsFilterLaunch> &launches, const QsFilterDesc *desc_dev, cudaStream_t st);

#endif
