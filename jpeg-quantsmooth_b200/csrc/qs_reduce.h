/* qs_reduce.h - the reduce stage of jpegqs_cuda_pixels_batch_reduced (qs_reduce.cu): Pillow's
 * Image.reduce (libImaging/Reduce.c) of an 8-bit HWC picture, byte for byte, and the planning of
 * Image.resize(..., reducing_gap=) and Image.thumbnail around it. */
#ifndef QS_REDUCE_H
#define QS_REDUCE_H

#include <cuda_runtime.h>
#include <stdint.h>
#include "qs_resize.h"

/* The largest cell (fx * fy samples) the reduce takes: Reduce.c's multiplier divides by the int
 * product 256 * n, which must stay below 2^31; below it the 32-bit sum cannot overflow either. */
#define QS_REDUCE_MAX_CELL (1 << 23)

/* One picture's reduce as the host planned it: the box (left, top, box_w x box_h) of the source
 * picture in fx x fy cells, out_w = ceil(box_w / fx) x out_h = ceil(box_h / fy).  fx = fy = 1: none. */
struct QsReducePlan {
	int32_t fx, fy, left, top, box_w, box_h, out_w, out_h;
};

/* One picture's reduce on the device (or in the host model, with host pointers). */
struct QsReduceDesc {
	const uint8_t *src;          /* the picture, HWC, src_w pixels of ch bytes a row */
	uint8_t *out;                /* out_h x out_w x ch */
	int32_t src_w, left, top, box_w, box_h, fx, fy, ch, out_w, out_h;
	uint32_t blk;                /* the picture's first block in the launch */
};

/* Pillow's Image.resize(out_w x out_h, filter, box, reducing_gap = gap) of a pic_w x pic_h picture,
 * gap 0 meaning None: the reduce over _get_safe_box (rd.fx = rd.fy = 1 when there is none) and the
 * resize of the reduced picture from the shifted float box (qs_resize_plan_box).  The plans count from
 * the picture's top-left corner.  Returns NULL, or why the picture cannot be taken (a cell of
 * QS_REDUCE_MAX_CELL samples or more; a picture more than 100 times taller than wide, which Pillow
 * resizes vertically first). */
const char *qs_reduced_plan(int pic_w, int pic_h, const double box[4], int out_w, int out_h, int filter, double gap,
		QsReducePlan &rd, QsResizePlan &rp);
/* Image.thumbnail's size (preserve_aspect_ratio) and draft scale for a width x height picture and a
 * bound_w x bound_h bound; loaded: the picture is already decoded (draft does nothing). */
void qs_thumbnail_geometry(int width, int height, int bound_w, int bound_h, double gap, int loaded, int *scale_denom,
		int *out_w, int *out_h);
void qs_reduce_desc(const QsReducePlan &rd, int src_w, int ch, QsReduceDesc &d);
/* numbers the blocks of the launch over the descriptors: sets each blk, returns the total */
uint32_t qs_reduce_number(QsReduceDesc *d, int n);
/* the launch over n descriptors in device memory */
cudaError_t qs_launch_reduce(const QsReduceDesc *desc_dev, int n, uint32_t blocks, cudaStream_t st);

#endif
