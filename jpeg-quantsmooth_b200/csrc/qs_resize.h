/* qs_resize.h - the crop-and-resize stage of jpegqs_cuda_pixels_batch_resized (qs_resize.cu): Pillow's
 * convolution resize (Resample.c) of an 8-bit HWC picture, byte for byte. */
#ifndef QS_RESIZE_H
#define QS_RESIZE_H

#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include "../../include/jpegqs_cuda.h"

/* One picture's resize as the host planned it.  tab holds four int32 tables back to back:
 *   hb [out_w][2]      the horizontal pass: first source column (in the crop) and tap count
 *   hk [out_w][ksh]    its weights, 22 fractional bits
 *   vb [out_h][2]      the vertical pass: first intermediate row and tap count
 *   vk [out_h][ksv]    its weights
 * The horizontal pass makes mid_h rows of out_w pixels: only the rows the vertical pass reads (Pillow's
 * ybox_first .. ybox_last of the crop).  top is the picture row of the first of them, and vb counts
 * from it. */
struct QsResizePlan {
	int32_t left, top, out_w, out_h, mid_h, ksh, ksv;
	std::vector<int32_t> tab;
};

/* One picture's resize on the device (or in the host model, with host pointers). */
struct QsResizeDesc {
	const uint8_t *src;          /* the picture, HWC, src_w pixels of ch bytes a row */
	uint8_t *mid, *out;          /* the intermediate, mid_h x out_w x ch; the output */
	const int32_t *tab;          /* QsResizePlan::tab */
	int32_t src_w, left, top, out_w, out_h, mid_h, ksh, ksv, ch;
	int32_t chw;                 /* 1: the output is ch planes (ch 3, JPEGQS_RENDER_CHW); 0: HWC */
	uint32_t hblk, vblk;         /* the picture's first block in each of the two launches */
};

/* the filter is one of JPEGQS_RESIZE_LANCZOS .. JPEGQS_RESIZE_HAMMING */
int qs_resize_filter_ok(int filter);
/* the filter's support (Pillow's _filters_support) */
double qs_resize_support(int filter);
/* Plans the crop box of a pic_w x pic_h picture resized to box.width x box.height.  Returns NULL, or
 * why the box does not fit (the crop outside the picture or empty; the output size outside 1..65535). */
const char *qs_resize_plan(int pic_w, int pic_h, const jpegqs_cuda_resize_box &box, int filter, QsResizePlan &rp);
/* Plans Pillow's Image.resize((out_w, out_h), filter, box) of the whole pic_w x pic_h picture from a float
 * box (left, top, right, bottom), as Pillow's C layer takes it.  For an integer box equal to the picture
 * the tables are qs_resize_plan's.  Returns NULL, or why the box does not fit. */
const char *qs_resize_plan_box(int pic_w, int pic_h, const float box[4], int out_w, int out_h, int filter, QsResizePlan &rp);
/* the host model of the two passes over src (src_w pixels of ch bytes a row) into out */
void qs_resize_run_model(const QsResizePlan &rp, const uint8_t *src, int src_w, int ch, int chw, uint8_t *out);
/* fills d's geometry from rp (the pointers are the caller's) */
void qs_resize_desc(const QsResizePlan &rp, int src_w, int ch, int chw, QsResizeDesc &d);
/* numbers the blocks of both launches over the descriptors: sets each hblk / vblk, returns the totals */
void qs_resize_number(QsResizeDesc *d, int n, uint32_t *hblocks, uint32_t *vblocks);
/* the two launches over n descriptors in device memory */
cudaError_t qs_launch_resize(const QsResizeDesc *desc_dev, int n, uint32_t hblocks, uint32_t vblocks, cudaStream_t st);

#endif
