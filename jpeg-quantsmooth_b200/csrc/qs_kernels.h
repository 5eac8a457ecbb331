/* launch wrappers implemented in qs_kernels.cu (internal, C++ linkage) */
#ifndef QS_KERNELS_H
#define QS_KERNELS_H
#include <cuda_runtime.h>
#include "qs_common.h"

size_t qs_smooth_smem_bytes(int diag, int wpg);
cudaError_t qs_smooth_configure(void);
cudaError_t qs_set_chunks(const QsChunk *chunks, int n);
cudaError_t qs_launch_idct_pass(const QsJob *jobs_dev, int njobs, int total_tiles, int mode,
		int *bad_flags, cudaStream_t st);
cudaError_t qs_launch_smooth(const QsJob *jobs_dev, int njobs, int total_tiles, const float *tables_dev,
		int *tile_counter, int flags, int clamp_out, int num_sms, int sync, int wpg, const int *bad, cudaStream_t st);
cudaError_t qs_launch_lowq(const QsJob *jobs_dev, int njobs, int total_tiles, int flags, int clamp_out,
		const int *bad, cudaStream_t st);
cudaError_t qs_launch_stop_fixup(const QsJob *jobs_dev, int njobs, const int *bad, cudaStream_t st);
cudaError_t qs_launch_xchg(const QsXchgPush *push, const QsXchgPull *pull, cudaStream_t st);
cudaError_t qs_launch_scale_clamp(int16_t *coef, size_t n, const QsQuantDev *qd, int dequant, int clamp,
		cudaStream_t st);
cudaError_t qs_launch_downsample(const uint8_t *src, int sstride, int w, int h, uint8_t *dst, int dstride,
		int w2, int h2, int ws, int hs, int src_row0, int dst_row_first, int dst_rows, int h1_total,
		cudaStream_t st);
cudaError_t qs_launch_upsample(const uint8_t *C, const uint8_t *Yd, int cstride, const uint8_t *Yf, int ystride,
		uint8_t *out, int ostride, int w1, int h1, int ws, int hs, int ww, int hh, int oy0, cudaStream_t st);
cudaError_t qs_launch_fdct_plane(const uint8_t *px, int pstride, int16_t *coef, int W, int H, cudaStream_t st);
cudaError_t qs_launch_render_rgb(const uint8_t *const *planes, const int *strides, const int *cw, const int *ch,
		const int *hs, const int *vs, int ncomp, int width, int height, int ycc, uint8_t *rgb, cudaStream_t st);
extern "C" int qs_host_orig_coef(int c, int q);
/* control data without the copy engines (see qs_kernels.cu) */
#define QS_JOB_PACK 48
cudaError_t qs_store_jobs(QsJob *dst, const QsJob *jobs_host, int n, cudaStream_t st);
cudaError_t qs_copy_flags(const int *src_dev, int *dst_mapped, int n, cudaStream_t st);
#define QS_QUANT_PACK 21
cudaError_t qs_store_quant(QsQuantDev *dst, const QsQuantDev *q_host, int n, cudaStream_t st);
/* per image of a stream-ordered run (qs_cuda.cu run_async): what its status is made of */
typedef struct {
	int32_t flag0;          /* slot of component 0 in the run's out-of-range flags */
	uint16_t iter_mask;     /* bit ci: component ci took part in the iterations */
	uint8_t host_stop;      /* a quant value >= 0x800 stopped it (quantsmooth.h:2504) */
	uint8_t kept;           /* the full-resolution luma plane was kept for UPSAMPLE_UV */
} QsStatusImg;
typedef struct { QsStatusImg img[QS_MAX_JOBS]; } QsStatusPack;
cudaError_t qs_launch_async_status(const QsStatusPack *p, int n, const int *flags, int2 *status, cudaStream_t st);

/* per image of a stream-ordered render (qs_cuda.cu render_async); tiles of QS_RENDER_TW x
 * QS_RENDER_TH output pixels, counted row by row from the image's tile_begin */
#define QS_RENDER_TW 128
#define QS_RENDER_TH 64
typedef struct {
	const int16_t *coef[3];      /* components 0..2 (1 and 2 unused for a grey image) */
	const int16_t *coef_up[2];   /* up-sampled chroma at component 0's geometry, or NULL */
	uint8_t *out;
	int32_t width, height, tile_begin;
	int32_t wblk[3], cw[3], ch[3];   /* cw / ch: libjpeg's downsampled_width / downsampled_height */
	uint8_t hs[3], vs[3];        /* expansion factors max_samp / samp */
	uint8_t ncomp, ycc;
	uint8_t up_mode;             /* 0: coef, 1: coef_up (host flag), 2: status[i].upsampled decides */
	uint8_t lss;                 /* scale_denom > 1: bits 2c..2c+1 hold log2 of component c's DCT scaled
	                                size; width, height, cw, ch, hs and vs are then the scaled ones */
	uint8_t orient;              /* 1..8: EXIF orientation of the output (include/jpegqs_cuda.h); width and
	                                height stay the unoriented picture's, out is H x W for 5..8 */
	uint16_t q[3][64];           /* multipliers: the raw quant table where it de-quantizes, else ones */
} QsRenderImg;
#define QS_RENDER_PACK 60
/* the descriptor of a 4-component (CMYK or YCCK) image: QsRenderImg's fields for four components, without
 * coef_up and up_mode (UPSAMPLE_UV never applies to these); lss holds four 2-bit fields */
typedef struct {
	const int16_t *coef[4];
	uint8_t *out;
	int32_t width, height, tile_begin;
	int32_t wblk[4], cw[4], ch[4];
	uint8_t hs[4], vs[4];
	uint8_t ncomp;               /* 4 */
	uint8_t ycc;                 /* 1: YCCK (components 0..2 YCbCr, libjpeg's ycck_cmyk_convert), 0: CMYK */
	uint8_t lss, orient;
	uint16_t q[4][64];
} QsRenderImg4;
#define QS_RENDER_PACK4 52
/* store modes of the render kernel: the two public layouts, and one byte per pixel for 1-component
 * images (qs_render_images' grey store) */
#define QS_RENDER_HWC 0
#define QS_RENDER_CHW 1
#define QS_RENDER_GREY 2
/* colour conversions of the render (Pillow's Image.convert of the decoded picture):
 *   NONE      the file's own colour: RGB for 3 components, the sample for grey (the existing kernels)
 *   L         Pillow's rgb2l of that RGB pixel; GREY store
 *   CMYK_RGB  4 components: Pillow's CMYK;I decode then cmyk2rgb (YCCK through ycck_cmyk_convert first)
 *   CMYK_L    4 components: rgb2l of CMYK_RGB's pixel; GREY store */
#define QS_CONV_NONE 0
#define QS_CONV_L 1
#define QS_CONV_CMYK_RGB 2
#define QS_CONV_CMYK_L 3
/* status: the launch's first image's {stop, upsampled}, or NULL when no image has up_mode 2;
 * scale_denom: 1, 2, 4 or 8; an orient outside 1..8 gives cudaErrorInvalidValue */
/* the render kernels' opt-in to the dynamic shared memory of orientations 5..8 (once per device) */
cudaError_t qs_render_configure(void);
/* conv: QS_CONV_NONE (any store) or QS_CONV_L (QS_RENDER_GREY) */
cudaError_t qs_launch_render_async(const QsRenderImg *imgs, int n, int tiles, const int2 *status, int store,
		int scale_denom, cudaStream_t st, int conv = QS_CONV_NONE);
/* 4-component images, n <= QS_RENDER_PACK4: conv QS_CONV_CMYK_RGB (HWC or CHW) or QS_CONV_CMYK_L (GREY) */
cudaError_t qs_launch_render4_async(const QsRenderImg4 *imgs, int n, int tiles, int store, int conv, int scale_denom,
		cudaStream_t st);
/* the same render of one image on the calling thread: host coefficient and output pointers, up_mode 0
 * or 1 */
void qs_render_host(const QsRenderImg *im, int store, int scale_denom, int conv = QS_CONV_NONE);
void qs_render4_host(const QsRenderImg4 *im, int store, int scale_denom, int conv);

#endif
