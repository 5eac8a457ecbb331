/*
 * jpegqs_cuda.h - C ABI of the H100 (sm_90a) back end of libjpegqs.
 *
 * This is the boundary between the libjpeg-facing host code (csrc/do_quantsmooth.c, which
 * keeps the reference's own entry points of libjpegqs.h) and the CUDA implementation.  It
 * occupies the slot of the reference's per-ISA workers do_quantsmooth_{base,sse2,avx2,avx512}
 * (reference libjpegqs.c:38-58, selected at libjpegqs.c:80-156): plain pointers and sizes,
 * no libjpeg types, no C++/torch types.  Every entry point cites the reference code it
 * replaces.  There is NO CPU fallback behind these calls: without a usable CUDA device they
 * fail with a negative return code.
 *
 * Layouts
 *   coefficients  int16 [hblk][wblk][64], natural (row-major) order inside a block - exactly
 *                 libjpeg's JBLOCKROW rows laid end to end (jpeglib.h JBLOCK / JCOEF).
 *   quant         the raw UINT16 quantval[64] of the component's JQUANT_TBL.
 */
#ifndef JPEGQS_CUDA_H
#define JPEGQS_CUDA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define JPEGQS_CUDA_MAX_COMP 10        /* libjpeg MAX_COMPONENTS */

/* error codes (all negative); >= 0 return values are the reference's `stop` value */
#define JPEGQS_ERR_CUDA  (-1)          /* CUDA runtime failure, see jpegqs_cuda_last_error */
#define JPEGQS_ERR_ARG   (-2)          /* malformed arguments */
#define JPEGQS_ERR_UNSUPPORTED (-3)    /* a knob of a measurement build asked of the shipped library */
#define JPEGQS_ERR_TIMEOUT (-4)        /* sharded run: a peer rank did not answer (see last_error) */

typedef struct jpegqs_cuda_ctx jpegqs_cuda_ctx;

/* One colour component as do_quantsmooth sees it: fields of jpeg_component_info that the
 * reference reads at quantsmooth.h:2484-2494 plus its coefficient array. */
typedef struct {
	int16_t *coef;          /* in: quantized; out: de-quantized + smoothed (in place)     */
	uint32_t wblk, hblk;    /* width_in_blocks, height_in_blocks                          */
	int32_t h_samp, v_samp; /* h_samp_factor, v_samp_factor                               */
	int32_t has_qtbl;       /* 0 when compptr->quant_table == NULL (component skipped)    */
	uint16_t quant[64];     /* raw quantval; overwritten with 1 on return (2851-2859)     */
	int16_t *coef_up;       /* out, comps 1..2 only: luma-sized array filled when
	                           UPSAMPLE_UV replaces the chroma arrays (2691-2752); may be
	                           NULL when UPSAMPLE_UV cannot trigger                        */
	/* Host entry points only - libjpeg's own layout: hblk pointers to block rows of wblk*64
	 * coefficients each, rows not necessarily adjacent (access_virt_barray, quantsmooth.h:
	 * 2592-2594).  When rows != NULL it replaces coef (which may be NULL), rows_up likewise
	 * replaces coef_up: the library gathers the rows into its pinned staging memory band by band
	 * on worker threads, overlapped with the uploads, and scatters the results back the same
	 * way.  The row memory must stay valid and untouched by the caller during the call. */
	int16_t **rows;
	int16_t **rows_up;
} jpegqs_cuda_comp;

typedef struct {
	int32_t ncomp;
	int32_t is_ycbcr;                   /* jpeg_color_space == JCS_YCbCr                   */
	uint32_t image_width, image_height;
	jpegqs_cuda_comp comp[JPEGQS_CUDA_MAX_COMP];
	int32_t upsampled;                  /* out: 1 = comps 1,2 now live in coef_up at the
	                                       luma geometry with 1x1 sampling (2835-2849)     */
} jpegqs_cuda_image;

typedef int (*jpegqs_cuda_progress_fn)(void *userdata, int cur, int max);

/* ---- context -------------------------------------------------------------------------- */
/* device < 0: the current CUDA device.  Returns 0 or a negative error code. */
int jpegqs_cuda_create(int device, jpegqs_cuda_ctx **out);
void jpegqs_cuda_destroy(jpegqs_cuda_ctx *ctx);
const char *jpegqs_cuda_last_error(const jpegqs_cuda_ctx *ctx);   /* ctx may be NULL */
const char *jpegqs_cuda_device_name(const jpegqs_cuda_ctx *ctx);
/* device time (CUDA events) of the kernels of the last run_* call, milliseconds */
float jpegqs_cuda_last_device_ms(const jpegqs_cuda_ctx *ctx);
/* number of kernel launches issued by the last run_* call */
int jpegqs_cuda_last_launches(const jpegqs_cuda_ctx *ctx);

/* optional per-kernel timing of the following run_* calls (CUDA event pairs around every
 * IDCT-pass and smoothing-pass launch, on the stream they are launched on); the sums are
 * read back with jpegqs_cuda_kernel_stats after the call.  Measurement aid for bench.py. */
void jpegqs_cuda_set_profiling(jpegqs_cuda_ctx *ctx, int on);
void jpegqs_cuda_kernel_stats(const jpegqs_cuda_ctx *ctx, float *idct_ms, int *idct_launches,
		float *smooth_ms, int *smooth_launches);

/* knobs for tuning runs and tests; results are bit-identical for every setting.
 * key 1: maximum coefficients per accumulation chunk (1..4, default 4)
 * key 5: uniform-quant chunks share t and d*t (default 1)
 * key 6: slab-pipelined upload / download in the host entry points (default 1)
 * key 7: blocks per slab wave for key 6; 0 = SM count x resident warps x 32 (tests force small values)
 * key 8: the two edge coefficients of an anti-diagonal ride along with up to two of its full
 *        coefficients in one "mixed" chunk instead of forming their own
 * key 9: entropy-coded bytes per decode subsequence of jpegqs_cuda_decode_async (>= 32, default
 *        512; tests force small values so that every file crosses many subsequence boundaries)
 * keys 0, 2 (lock-step level, warps per sub-partition) only exist in the measurement build
 * (make -C csrc experiments); the shipped library accepts their default values and answers
 * JPEGQS_ERR_UNSUPPORTED otherwise.  key 3: retired, ignored.  key 4: retired (a packed FP32x2
 * path); every build accepts 0 only. */
int jpegqs_cuda_set_tuning(jpegqs_cuda_ctx *ctx, int key, int value);

/* pinned host memory for coefficient arrays: the copy engines read / write it directly.  Plain
 * malloc'd memory (flat or as block-row tables, see jpegqs_cuda_comp.rows) works too and goes
 * through the context's pinned staging buffer, which is kept between calls (grow-only).
 * Environment: JPEGQS_IO_THREADS = threads used for that gather / scatter (default: up to 8). */
void *jpegqs_cuda_host_alloc(size_t bytes);
void jpegqs_cuda_host_free(void *p);

/* ---- whole-image entry points: the body of do_quantsmooth (quantsmooth.h:2404-2878) ----
 * flags/niter/progprec/progress/userdata = jpegqs_control_t fields (libjpegqs.h:41-45).
 * With progress == NULL independent components are processed in the same kernel launches;
 * with a callback components run one after another so the callback sequence (cur, max) is
 * the reference's (quantsmooth.h:2656-2664).
 * Return: the reference's `stop` (0 = done, non-zero = stopped early) or a negative error. */
int jpegqs_cuda_run_host(jpegqs_cuda_ctx *ctx, jpegqs_cuda_image *img, int flags, int niter,
		int progprec, jpegqs_cuda_progress_fn progress, void *userdata);
/* same, but comp[].coef / coef_up are DEVICE pointers; stream = cudaStream_t or NULL */
int jpegqs_cuda_run_device(jpegqs_cuda_ctx *ctx, jpegqs_cuda_image *img, int flags, int niter,
		int progprec, jpegqs_cuda_progress_fn progress, void *userdata, void *stream);
/* n independent images in shared launches (no progress callback); host or device pointers.
 * ret[i] receives each image's stop value.  Returns 0 or a negative error. */
int jpegqs_cuda_run_batch(jpegqs_cuda_ctx *ctx, int nimages, jpegqs_cuda_image *imgs, int flags,
		int niter, int on_device, int *ret, void *stream);

/* ---- stream-ordered, graph-capturable run over device buffers ---------------------------
 * What jpegqs_cuda_run_batch(on_device = 1) computes, for a caller that keeps its data on the GPU
 * and its host thread free:
 *   - comp[].coef / coef_up are DEVICE pointers on the context's device; rows / rows_up must be
 *     NULL.  No progress callback.
 *   - Nothing is read back and nothing waits: the call returns once all its work is enqueued on
 *     stream (NULL: the context's stream).  status_dev[i] (device memory) receives image i's
 *     {stop, upsampled} on the stream - the values run_device returns and puts in img->upsampled;
 *     img->upsampled is left at 0 here.  quant[] is set to 1 on return, as by the other entry
 *     points (it does not depend on the data).
 *   - Argument errors change nothing: every check runs before the first enqueue and a failed one
 *     returns JPEGQS_ERR_ARG with nothing enqueued.  Checked: workspace too small or not 256-byte
 *     aligned, status_dev NULL, malformed geometry (ncomp outside 1..10, a sampling factor outside
 *     1..4, a non-empty component without coef, unequal chroma components where JOINT_YUV /
 *     UPSAMPLE_UV down-sample the luma - whatever niter is), and coef_up missing where UPSAMPLE_UV
 *     can trigger.  A CUDA error while enqueueing returns JPEGQS_ERR_CUDA.
 *   - All per-call device state lives in the workspace: sample planes, the down-sampled luma, the
 *     up-sampled chroma planes, quant constants, job lists, out-of-range flags and the tile
 *     counter.  The call writes all of it earlier in its own stream work than anything reads it, so
 *       . the next call on the same stream may reuse the workspace without clearing it;
 *       . two calls on different streams of one context, with separate workspaces, may be in
 *         flight together;
 *       . a CUDA graph captured around the call replays correctly: a replay re-runs the call on
 *         the current contents of the same coefficient, coef_up, workspace and status buffers,
 *         with the geometry, quant tables, flags and niter fixed at capture.
 *   - Host memory is released at return: job lists and quant constants travel as kernel
 *     parameters, and the call reads nothing of imgs afterwards.
 *   - No cudaMalloc, no synchronisation, no event query or record: the call is legal under
 *     cudaStreamCaptureModeGlobal (what torch.cuda.graph uses).  So jpegqs_cuda_last_device_ms
 *     keeps its value and profiling is ignored; jpegqs_cuda_last_launches counts the launches.
 *   - Batches of more than 1024 components run as sub-batches one after another on the stream.
 *   - As everywhere: one calling thread per context at a time.
 * Returns 0 or a negative error. */
typedef struct { int32_t stop, upsampled; } jpegqs_cuda_status;

/* Device bytes of workspace jpegqs_cuda_run_async needs for these images and flags (host-only, no
 * device needed; checks the geometry as jpegqs_cuda_run_async does, not the pointers).  With
 * A(x) = x rounded up to a multiple of 256 and C = the number of components of all images:
 *   168192 + A(1544 * C)                             flags + tile counter, job lists, quant constants
 *   + for every component:  A(jpegqs_cuda_plane_bytes(wblk, hblk))       its sample plane
 *   + for every image whose chroma JOINT_YUV / UPSAMPLE_UV feed from a down-sampled luma (YCbCr,
 *     >= 3 components, components 1 and 2 sampled 1x1, component 0 not):
 *       A(jpegqs_cuda_plane_bytes(comp[1].wblk, comp[1].hblk))          the down-sampled luma
 *       + with UPSAMPLE_UV: 2 * A(comp[0].wblk * comp[0].hblk * 64)     the up-sampled chroma   */
int jpegqs_cuda_async_workspace_bytes(int nimages, const jpegqs_cuda_image *imgs, int flags, size_t *bytes);
int jpegqs_cuda_run_async(jpegqs_cuda_ctx *ctx, int nimages, jpegqs_cuda_image *imgs, int flags, int niter,
		void *workspace, size_t workspace_bytes, jpegqs_cuda_status *status_dev, void *stream);

/* ---- stream-ordered, graph-capturable render of device-resident images to 8-bit RGB -------
 * What libjpeg's jpeg_read_scanlines gives for these coefficients with out_color_space JCS_RGB,
 * JDCT_ISLOW and fancy up-sampling (the pixels jpegqs_cuda_render_rgb computes), for a caller
 * whose coefficients are on the GPU - typically right after jpegqs_cuda_run_async, in the same
 * stream or CUDA graph.  One fused kernel per batch: IDCT, up-sampling and colour conversion
 * without any sample plane in device memory and without a workspace.
 *   - Inputs.  comp[].coef / coef_up are DEVICE pointers on the context's device, 16-byte aligned
 *     (blocks are read as 16-byte vectors); rows / rows_up must be NULL.  1 or 3 components: 3 are converted YCbCr -> RGB when is_ycbcr is set and
 *     copied otherwise, 1 is replicated to R = G = B (JCS_GRAYSCALE -> JCS_RGB).  Any other count,
 *     or sampling factors whose ratios are not integral (libjpeg cannot decode those either),
 *     returns JPEGQS_ERR_UNSUPPORTED with nothing enqueued.
 *   - Coefficients are only read.  A component with has_qtbl and a quant table that is not all
 *     ones (render_rgb's rule: still quantized) is de-quantized in registers, in int32 as libjpeg
 *     does, so a never-smoothed coefficient set decodes too; nothing is written back.  Component
 *     c's table applies to whichever array is read for it (after run_async all tables are ones).
 *   - Chroma source.  Components 1 and 2 come from coef_up, at component 0's geometry with 1x1
 *     sampling, when the image is up-sampled, and from coef otherwise:
 *       . status_dev != NULL: up-sampled means status_dev[i].upsampled != 0, read on the device,
 *         for images whose two coef_up pointers are non-NULL; other images always read coef.  So
 *         one graph may hold run_async followed by this call, and a replay in which an image
 *         stops (and so is not up-sampled) renders it from coef.
 *       . status_dev == NULL: imgs[i].upsampled decides (callers of run_device and run_batch).
 *   - Output.  out_dev[i]: image_width * image_height * 3 bytes of device memory at any byte
 *     alignment (a slice of a batched [N, H, W, 3] tensor works), in layout JPEGQS_RENDER_HWC or
 *     JPEGQS_RENDER_CHW.
 *   - Argument errors change nothing: every check runs before the first enqueue and a failed one
 *     returns JPEGQS_ERR_ARG with nothing enqueued.  Checked: out_dev or an entry of it NULL, a
 *     coef pointer NULL (or a coef_up one for a host-flagged up-sampled image), a coef or coef_up
 *     pointer not 16-byte aligned, rows / rows_up set, a sampling factor outside 1..4, a component whose blocks do not cover its samples
 *     (wblk * 8 < cw or hblk * 8 < ch, with cw = ceil(image_width * h_samp / max_h_samp) and ch
 *     likewise, libjpeg's downsampled_width / height), and an unknown layout.
 *   - The stream rules of run_async: no cudaMalloc, synchronisation, event record or query, and no
 *     context memory (per-image descriptors and quant tables travel as kernel parameters), so the
 *     call is legal under cudaStreamCaptureModeGlobal and may be in flight with run_async or
 *     render_async calls on other streams of the same context.  Host structs may be freed at
 *     return.  jpegqs_cuda_last_launches counts its launches; batches larger than one launch's
 *     parameter space (60 images) run as several launches, one after another on the stream.
 * Returns 0 or a negative error. */
#define JPEGQS_RENDER_HWC 0   /* R,G,B interleaved per pixel: libjpeg's JCS_RGB scanlines      */
#define JPEGQS_RENDER_CHW 1   /* three planes R, G, B of image_width * image_height bytes each */
int jpegqs_cuda_render_async(jpegqs_cuda_ctx *ctx, int nimages, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_status *status_dev, int layout, uint8_t *const *out_dev, void *stream);

/* ---- the same render at 1/2, 1/4 or 1/8 size: libjpeg's scaled decode -----------------------
 * jpegqs_cuda_render_async is this call with scale_denom 1; everything above holds, except:
 *   - Output.  out_dev[i]: ceil(image_width / d) * ceil(image_height / d) * 3 bytes, d = scale_denom.
 *   - Pixels.  What jpeg_read_scanlines gives for the coefficients with scale_num 1, scale_denom d,
 *     JDCT_ISLOW, do_fancy_upsampling TRUE and JCS_RGB output.  The image never exists at full size:
 *       . each component gets libjpeg's DCT scaled size (jpeg_calc_output_dimensions): 8 / d, doubled
 *         while the sampling ratios allow, so chroma is scaled up by its IDCT rather than up-sampled
 *         where possible (4:2:0 at 1/2: luma 4x4, chroma 8x8, no up-sampling);
 *       . blocks of scaled size 4, 2 and 1 go through libjpeg's reduced IDCTs (jidctred.c
 *         jpeg_idct_4x4 / 2x2 / 1x1), size 8 through the islow IDCT;
 *       . downsampled_width / height and the up-sampling ratios are computed at the scaled sizes;
 *         fancy up-sampling is used where libjpeg uses it: not at d = 8 (smallest scaled size 1), and
 *         h2v1 / h2v2 replicate when the scaled downsampled_width is 2 or less.
 *   - Checked as well: scale_denom outside {1, 2, 4, 8} returns JPEGQS_ERR_ARG with nothing enqueued,
 *     and the blocks must cover the samples at the scaled geometry (wblk * size >= downsampled_width).
 * Returns 0 or a negative error. */
int jpegqs_cuda_render_scaled_async(jpegqs_cuda_ctx *ctx, int nimages, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_status *status_dev, int layout, int scale_denom, uint8_t *const *out_dev, void *stream);

/* jpegqs_cuda_render_scaled_async's algorithm on the calling thread, for one image (host-only, no
 * device needed): the same reduced IDCTs, up-sampling and colour conversion.  comp[].coef / coef_up
 * are HOST arrays; upsampled != 0 reads components 1 and 2 from coef_up, as a host-flagged up-sampled
 * image.  out: ceil(image_width / d) * ceil(image_height / d) * 3 bytes in layout HWC or CHW (a grey
 * image gives R = G = B).  Returns 0, JPEGQS_ERR_ARG (NULL img or out, unknown layout, scale_denom
 * outside {1, 2, 4, 8}, the geometry checks of render_async) or JPEGQS_ERR_UNSUPPORTED (what
 * render_async does not render); jpegqs_cuda_last_error(NULL) says why. */
int jpegqs_cuda_render_model(const jpegqs_cuda_image *img, int upsampled, int layout, int scale_denom, uint8_t *out);

/* ---- EXIF orientation ---------------------------------------------------------------------------
 * Orientation o (1..8) is the transform Pillow's ImageOps.exif_transpose applies.  The oriented picture
 * is W' x H' (W' = H, H' = W for o = 5..8), and its pixel (x', y') is pixel (x, y) of the W x H stored one:
 *     o  Pillow's Image.transpose   (x, y)
 *     1  (none)                     (x', y')
 *     2  FLIP_LEFT_RIGHT            (W-1-x', y')
 *     3  ROTATE_180                 (W-1-x', H-1-y')
 *     4  FLIP_TOP_BOTTOM            (x', H-1-y')
 *     5  TRANSPOSE                  (y', x')
 *     6  ROTATE_270                 (y', H-1-x')
 *     7  TRANSVERSE                 (W-1-y', H-1-x')
 *     8  ROTATE_90                  (W-1-y', x')
 *
 * jpegqs_cuda_render_scaled_async with a host array of one orientation 1..8 per image (NULL: all 1,
 * which is render_scaled_async; render_async and render_scaled_async are this call with NULL).
 * out_dev[i] receives the oriented picture: W' x H' pixels in the layout (CHW planes W' x H'), the
 * same number of bytes.  The transform happens in the render's store, not as a second pass.  Same
 * stream rules (no allocation, no synchronisation, graph-capturable; the orientations are fixed at
 * capture).  A value outside 1..8 returns JPEGQS_ERR_ARG with nothing enqueued. */
int jpegqs_cuda_render_oriented_async(jpegqs_cuda_ctx *ctx, int nimages, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_status *status_dev, int layout, int scale_denom, const int32_t *orientation,
		uint8_t *const *out_dev, void *stream);

/* ---- colour conversion: Pillow's Image.convert("RGB") / convert("L") of the decoded picture ---------
 * mode JPEGQS_PIXELS_AS_FILE (0) is the file's own colour, the existing calls' behaviour: RGB for 3
 * components, one grey sample for 1, and 4 components are not rendered (JPEGQS_ERR_UNSUPPORTED).
 * JPEGQS_PIXELS_RGB (1) gives 3 channels and JPEGQS_PIXELS_L (2) gives 1, whatever the component count:
 *   - 1 component: RGB replicates the sample; L is the sample.
 *   - 3 components: RGB is the existing render; L is Pillow's rgb2l of it,
 *     (R * 19595 + G * 38470 + B * 7471 + 0x8000) >> 16 - not the file's Y plane.
 *   - 4 components: what Pillow decodes (libjpeg's JCS_CMYK output with raw mode CMYK;I, which inverts
 *     all four samples), then its cmyk2rgb: with nk = 255 - K, out = nk - MULDIV255(C, nk) per channel,
 *     MULDIV255(a, b) = (t = a * b + 128, ((t >> 8) + t) >> 8).  A YCCK file goes through libjpeg's
 *     ycck_cmyk_convert first (the YCbCr -> RGB of the 3-component render, inverted; K passes through).
 *     L is rgb2l of that RGB.
 * The conversion is per pixel, so it commutes with the orientation; the crop, the resize and the
 * compressor take the converted picture.  Colour space: libjpeg's default_decompress_parms rule, which
 * jpegqs_cuda_scan.jpeg_color_space gives: 4 components are CMYK without an Adobe marker or with transform
 * 0, and YCCK with any other transform. */
#define JPEGQS_PIXELS_AS_FILE 0
#define JPEGQS_PIXELS_RGB 1
#define JPEGQS_PIXELS_L 2

/* jpegqs_cuda_render_oriented_async with a colour conversion (render_oriented_async is this call with
 * color_space NULL and mode 0).  color_space: NULL, or one JCS_* value per image (jpeglib.h numbering:
 * GRAYSCALE 1, RGB 2, YCbCr 3, CMYK 4, YCCK 5) that decides the conversion in place of is_ycbcr; NULL
 * derives it from ncomp and is_ycbcr, 4 components being CMYK.  A value the image's component count cannot
 * have, or a mode other than the three above, returns JPEGQS_ERR_ARG with nothing enqueued.  out_dev[i]:
 * W' * H' * channels bytes (channels as above; mode 0: 3).  4-component images take 624-byte descriptors,
 * 52 per launch.  Same stream rules; graph-capturable. */
int jpegqs_cuda_render_mode_async(jpegqs_cuda_ctx *ctx, int nimages, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_status *status_dev, int layout, int scale_denom, const int32_t *orientation,
		const int32_t *color_space, int mode, uint8_t *const *out_dev, void *stream);

/* jpegqs_cuda_render_model with a colour space (a JCS_* value as above, or -1 to derive it as NULL does)
 * and a mode; out: W * H * channels bytes (mode 0: 3).  jpegqs_cuda_render_model is this call with -1 and
 * mode 0. */
int jpegqs_cuda_render_model_mode(const jpegqs_cuda_image *img, int color_space, int upsampled, int layout,
		int scale_denom, int mode, uint8_t *out);

/* Host-only, no device needed.  *orientation = the orientation ImageOps.exif_transpose(Image.open(f))
 * applies to file f, 1 for none - including every file where Pillow's getexif() raises.  The rules are
 * those of Pillow 12.2 (JpegImagePlugin, Image.getexif, Image.Exif.load, TiffImagePlugin
 * ImageFileDirectory_v2), not the EXIF specification's:
 *   - Segments: only those before the first SOS.  The first APP1 starting "Exif\0\0" is the EXIF
 *     block and later ones are appended without those 6 bytes; of the APP1s starting
 *     "http://ns.adobe.com/xap/1.0/\0" (XMP), the last one counts.
 *   - EXIF: leading "Exif\0\0"s are dropped; an empty block has no tags.  A TIFF header "II*\0",
 *     "MM\0*" (or the swapped "II\0*", "MM*\0") and IFD0 at its offset; any other header, a BigTIFF
 *     one or fewer than 8 bytes make getexif raise (1, XMP not read).  Of IFD0's 0x0112 entries the
 *     last one kept wins.  An entry of an unknown type or with count 0 is skipped; an entry cut short,
 *     or whose data lies past the block, ends the IFD and keeps the entries before it.
 *   - Value: the first value, as Pillow decodes the type, looked up in a dict of 2..8: SHORT, LONG,
 *     the signed integers, FLOAT / DOUBLE and (SIGNED) RATIONAL equal to one of them count (6, 6.0 and
 *     12/2 all give 6); BYTE, UNDEFINED and ASCII decode to bytes or str and give 1, as does any
 *     other number.
 *   - XMP, only when the EXIF has no 0x0112 entry: the first match of tiff:Orientation(="|>)([0-9]);
 *     its digit if 2..8, else 1.
 * Only [data, data + len) is read, whatever the offsets and counts say, and nothing past the first SOS
 * segment.  Returns 0, or JPEGQS_ERR_ARG for a file whose markers up to the first SOS the tool's reader
 * rejects (jpegqs_cuda_jpeg_parse's header walk; jpegqs_cuda_last_error(NULL) has the message). */
#define JPEGQS_ORIENT_FILE 0  /* in the batch calls' orientation arrays: the file's own orientation */
int jpegqs_cuda_jpeg_orientation(const uint8_t *data, size_t len, int32_t *orientation);

/* ---- JPEG files to quantized coefficients -----------------------------------------------------
 * The first stage of a device pipeline: JPEG bytes -> the coefficients jpeg_read_coefficients gives,
 * as [hblk][wblk][64] int16 arrays, exactly what jpegqs_cuda_run_async and jpegqs_cuda_render_async
 * take.  jpegqs_cuda_jpeg_parse reads the markers up to the first SOS on the host;
 * jpegqs_cuda_decode_async decodes the entropy-coded data on the GPU for the files parse accepts,
 * jpegqs_cuda_jpeg_read on host threads for all others.
 *
 * The scan a device decode needs: what is in force at the first SOS.  No libjpeg types. */
typedef struct {
	int32_t ncomp;                    /* components in the scan                                  */
	int32_t comp[4];                  /* frame component index of scan component k (MCU order)  */
	int32_t dc_tbl[4], ac_tbl[4];     /* table selectors (Td, Ta) of scan component k            */
	int32_t dc_present[4], ac_present[4];  /* 1 = table slot defined by a DHT before the SOS     */
	uint8_t dc_bits[4][17], dc_val[4][256];  /* DHT's BITS (index 1..16; 0 unused) and HUFFVAL  */
	uint8_t ac_bits[4][17], ac_val[4][256];
	uint32_t restart_interval;        /* DRI value in force, MCUs; 0 = no restart markers        */
	uint64_t entropy_offset;          /* byte offset of the first entropy-coded byte in the file */
	int32_t jpeg_color_space;         /* libjpeg's J_COLOR_SPACE guess (JCS_* values of jpeglib.h) */
	int32_t sof;                      /* 0xC0 / 0xC1 / 0xC2: the frame's SOF marker             */
} jpegqs_cuda_scan;

/* Host-only, no device needed.  Fills img (ncomp, is_ycbcr, image size; per component wblk, hblk,
 * sampling, has_qtbl, quant; coef / coef_up / rows / rows_up NULL) and scan from the markers before
 * the first SOS, with the marker walk of the jpegqs tool's reader.  Returns
 *   0                       the device decoder takes the file: SOF0 / SOF1, 8-bit samples, and the
 *                           first scan holds all 1-4 components;
 *   JPEGQS_ERR_UNSUPPORTED  img and scan filled, but only jpegqs_cuda_jpeg_read takes it (progressive
 *                           files, sequential files with more than one scan, Huffman tables libjpeg
 *                           would reject for a device decode: an all-ones code or a DC symbol > 15);
 *   JPEGQS_ERR_ARG          what the reader rejects (jpegqs_cuda_last_error(NULL) has its message). */
int jpegqs_cuda_jpeg_parse(const uint8_t *data, size_t len, jpegqs_cuda_image *img, jpegqs_cuda_scan *scan);
/* Host decode of any file the jpegqs tool reads (its reader: several threads, libjpeg-compatible
 * handling of damaged data) into img->comp[c].coef: HOST arrays [hblk][wblk][64] of the geometry
 * jpegqs_cuda_jpeg_parse reports.  Returns the number of warnings (recoverable damage, >= 0) or
 * JPEGQS_ERR_ARG (message in jpegqs_cuda_last_error(NULL)). */
int jpegqs_cuda_jpeg_read(const uint8_t *data, size_t len, const jpegqs_cuda_image *img);

/* Stream-ordered, graph-capturable decode of n files' entropy-coded data on the GPU.
 *   - Inputs.  data_dev[i]: DEVICE memory holding file i from its first byte, data_len[i] bytes long.
 *     imgs[i] / scans[i]: what jpegqs_cuda_jpeg_parse returned 0 for (the host structs are read during
 *     the call only).  The entropy-coded segment starts at scans[i].entropy_offset; the device finds
 *     its end, the first marker that is not RSTn (any marker when restart_interval is 0).  Bytes
 *     after it are ignored.
 *   - Output.  imgs[i].comp[c].coef: DEVICE pointers, 16-byte aligned, [hblk][wblk][64] int16:
 *     the quantized coefficients jpeg_read_coefficients gives, natural order - run_async's input.
 *     Blocks of the MCU padding (beyond wblk / hblk in an interleaved scan) are decoded and dropped.
 *     DC predictors are int and stored as (JCOEF), as libjpeg does.
 *   - Status.  status_dev[i] (device int32) is 0 when image i decoded cleanly, otherwise an OR of
 *     the JPEGQS_DECODE_* bits below.  status 0 => the coefficients equal jpeg_read_coefficients'.  A
 *     flagged image's coefficients are unspecified, but every write stays inside that image's arrays
 *     and every loop is bounded by the data length; the other images are not affected.
 *   - Stream features.  Accepted (status 0): FF fill bytes before the marker that ends the segment,
 *     restart intervals of any length up to 65535 (also the MCU count and more), any component
 *     identifiers and table slots, Huffman codes up to 16 bits.  Flagged (the host reader, which
 *     accepts them as libjpeg does, decodes these): FF fill bytes before an RSTn (the segment ends at
 *     the first FF, so RESTART | UNITS), and an interval's padding with 0-bits instead of 1-bits
 *     (UNITS, with TRUNCATED for a sequential scan).  tests/stream_files.py holds a file of each.
 *   - Argument errors change nothing: every check runs before the first enqueue and a failed one
 *     returns JPEGQS_ERR_ARG with nothing enqueued.  Checked: NULL pointers (imgs, scans, data_dev and
 *     its entries, data_len, status_dev, coef), a coef not 16-byte aligned, rows / rows_up set, a
 *     workspace too small or not 256-byte aligned, entropy_offset >= data_len, ncomp outside 1..4 or
 *     unequal to the scan's, scan components that are not a permutation of the frame's, selectors
 *     naming absent or invalid tables, sampling factors outside 1..4 or more than 10 blocks per MCU,
 *     and wblk / hblk other than libjpeg's width_in_blocks / height_in_blocks.  A CUDA error while
 *     enqueueing returns JPEGQS_ERR_CUDA.
 *   - The stream rules of run_async: no cudaMalloc, no synchronisation, no event record or query, no
 *     host memory read after return.  Huffman tables and per-image descriptors travel as kernel
 *     parameters.  Legal under cudaStreamCaptureModeGlobal: a replay decodes the current contents of
 *     the same data, coef, workspace and status buffers, with the headers (geometry, tables,
 *     restart interval, entropy offset) and data_len fixed at capture - so a captured graph decodes
 *     the next file of a stream of same-header files.  Two calls on different streams with separate
 *     workspaces may be in flight together.  jpegqs_cuda_last_launches counts the launches (ten per
 *     group of up to 8 images; larger batches run as several groups, one after another).
 *   - Workspace: all per-call device state (the unstuffed data, restart positions, per-subsequence
 *     decoder states and counts, the derived Huffman look-up tables).  With A(x) = x rounded up to a
 *     multiple of 256, L = data_len - entropy_offset, I = ceil(MCUs / restart_interval) (1 without
 *     restarts; MCUs = blocks for a one-component scan), the size is the sum over images of
 *       16384 + A(L + 8) + A(24 * ceil(L / 4096)) + 2 * A(4 * I) + A(96 * (floor(L / 32) + I))
 *     It does not depend on tuning key 9 (it is sized for the smallest value, 32).
 * Returns 0 or a negative error. */
#define JPEGQS_DECODE_BAD_CODE   1    /* a bit pattern that is no Huffman code of the table        */
#define JPEGQS_DECODE_TRUNCATED  2    /* a unit read past the end of its data / restart interval   */
#define JPEGQS_DECODE_RESTART    4    /* a restart marker missing, extra or out of sequence        */
#define JPEGQS_DECODE_AC_RUN     8    /* an AC coefficient placed past coefficient 63              */
#define JPEGQS_DECODE_UNITS     16    /* the data does not hold the image's number of MCUs         */
int jpegqs_cuda_decode_workspace_bytes(int n, const jpegqs_cuda_image *imgs, const jpegqs_cuda_scan *scans,
		const size_t *data_len, size_t *bytes);
int jpegqs_cuda_decode_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_scan *scans, const uint8_t *const *data_dev, const size_t *data_len,
		void *workspace, size_t workspace_bytes, int32_t *status_dev, void *stream);

/* ---- any scan script: progressive and multi-scan files ------------------------------------------
 * jpegqs_cuda_decode_async takes files with one interleaved sequential scan.  The calls below take
 * every file the jpegqs tool's reader takes - SOF0 / SOF1 / SOF2, Huffman, 8-bit samples, any scan
 * script of up to JPEGQS_MAX_SCANS scans - and give the coefficients jpeg_read_coefficients gives.
 *
 * One scan as the host marker walk found it.  No libjpeg types. */
#define JPEGQS_MAX_SCANS 64
typedef struct {
	int32_t ncomp;                    /* components in the scan (1 for progressive AC scans)     */
	int32_t comp[4];                  /* frame component index of scan component k (MCU order)  */
	int32_t dc_tbl[4], ac_tbl[4];     /* table selectors (Td, Ta) of scan component k            */
	int32_t Ss, Se, Ah, Al;           /* spectral selection and successive approximation; a
	                                   * sequential scan has 0, 63, 0, 0                         */
	int32_t sof;                      /* the frame's SOF marker: 0xC0 / 0xC1 / 0xC2              */
	int32_t dc_present[4], ac_present[4];  /* the Huffman tables in force at this SOS (a DHT may   */
	uint8_t dc_bits[4][17], dc_val[4][256];  /* sit between scans): BITS (index 1..16) and HUFFVAL */
	uint8_t ac_bits[4][17], ac_val[4][256];
	uint32_t restart_interval;        /* DRI in force at this SOS; MCUs (blocks when ncomp = 1)  */
	uint64_t offset;                  /* first entropy-coded byte of the scan                    */
	uint64_t end;                     /* the next marker that is not RSTn, or the file's end when none
	                                   * follows: the segment is [offset, end)                    */
} jpegqs_cuda_scan_rec;

/* Host-only.  Walks every marker of the file without decoding entropy-coded data: fills img as
 * jpegqs_cuda_jpeg_parse does and scans[0 .. *nscans) (cap entries; *nscans is set whenever the
 * walk succeeds, also when it exceeds cap).  Returns
 *   0                       the file's scans are all in scans[] and jpegqs_cuda_decode_scans_async
 *                           takes them;
 *   JPEGQS_ERR_UNSUPPORTED  more scans than cap or JPEGQS_MAX_SCANS, a scan without a single
 *                           entropy-coded byte (a file cut at an SOS), a selected Huffman table libjpeg
 *                           would reject (an all-ones code, a DC symbol > 15), or a first scan
 *                           (Ah = 0) after an AC refinement scan of the same component whose band
 *                           overlaps it (not a T.81 scan script): jpegqs_cuda_jpeg_read takes these;
 *   JPEGQS_ERR_ARG          what the reader rejects (message in jpegqs_cuda_last_error(NULL)),
 *                           a scan using an undefined table included. */
int jpegqs_cuda_jpeg_parse_scans(const uint8_t *data, size_t len, jpegqs_cuda_image *img,
		jpegqs_cuda_scan_rec *scans, int cap, int *nscans);

/* Stream-ordered, graph-capturable decode of n files of any scan script on the GPU.
 *   - Inputs.  data_dev[i] / data_len[i] as for decode_async; imgs[i] and scans[i][0 .. nscans[i])
 *     what jpegqs_cuda_jpeg_parse_scans returned 0 for (host structs, read during the call only).
 *   - Output.  imgs[i].comp[c].coef: DEVICE pointers, 16-byte aligned, [hblk][wblk][64] int16.  The
 *     call zeroes them first (coefficients no scan codes are 0), so a replay rewrites them whole.
 *   - Status.  status_dev[i]: 0 or an OR of the JPEGQS_DECODE_* bits; status 0 => the coefficients
 *     equal jpeg_read_coefficients'.  Every write stays inside image i's arrays.
 *   - Schedule, per group of images (up to 16 images and 512 scans): zero the arrays; one byte pass
 *     (unstuffing, RSTn) over every scan; every sequential, DC first and AC first scan through one set
 *     of the speculative-subsequence launches of decode_async (in an AC first scan an end-of-band run
 *     is one decoder step that counts all its blocks; a run that outlives its restart interval is cut
 *     there); every DC refinement scan in one launch (one thread per block); AC refinement scans one
 *     launch per level, one warp per restart interval.  The level of an AC refinement scan is one
 *     more than the highest among the earlier AC refinement scans of its component whose bands
 *     overlap.  Within a restart interval (the whole scan without restart markers) an AC refinement
 *     scan is decoded serially: a file without restart markers decodes each such scan on one thread.
 *   - Argument errors change nothing: every check runs before the first enqueue.  Checked besides
 *     decode_async's image checks: nscans[i] outside 1..JPEGQS_MAX_SCANS, a scan's components not
 *     distinct frame components, Ss / Se / Ah / Al outside T.81's ranges, an AC scan of several
 *     components, offset / end outside data_len, a table the scan decodes with absent or invalid.
 *   - The stream rules of decode_async: no allocation, synchronisation or event use; descriptors and
 *     Huffman tables travel as kernel parameters (a store kernel per 24 scans writes them to the
 *     workspace).  Under graph capture every scan's header, position, tables and restart interval
 *     and data_len are fixed at capture: a replay decodes the current bytes of the same buffers, so
 *     it decodes a file whose headers and scan positions are identical to the captured one's.
 *     jpegqs_cuda_last_launches counts the launches.
 *   - Workspace.  With A(x) = x rounded up to a multiple of 256, per scan L = end - offset and I =
 *     ceil(MCUs / restart_interval) (1 without restarts; MCUs = blocks for a one-component scan), the
 *     size is the sum over images and scans of
 *       16384 + A(L + 8) + A(24 * ceil(L / 4096)) + 2 * A(4 * I) + S
 *     with S = A(96 * (floor(L / 32) + I)) for sequential and first scans and S = 0 for refinement
 *     scans.  It does not depend on tuning key 9.
 * Returns 0 or a negative error. */
int jpegqs_cuda_decode_scans_workspace_bytes(int n, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_scan_rec *const *scans, const int *nscans, const size_t *data_len, size_t *bytes);
int jpegqs_cuda_decode_scans_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_scan_rec *const *scans, const int *nscans, const uint8_t *const *data_dev,
		const size_t *data_len, void *workspace, size_t workspace_bytes, int32_t *status_dev, void *stream);
/* jpegqs_cuda_decode_scans_async's algorithm on one CPU thread, for one file: the same byte pass, the
 * same subsequences of sub_bytes (>= 32) bytes, the same step decoders, placement, refinement
 * decoders and scan order.  img->comp[c].coef are HOST arrays (zeroed by the call).  *status
 * receives the JPEGQS_DECODE_* bits. */
int jpegqs_cuda_decode_scans_model(const jpegqs_cuda_image *img, const jpegqs_cuda_scan_rec *scans, int nscans,
		const uint8_t *data, size_t data_len, int sub_bytes, int32_t *status);

/* ---- quantized coefficients to JPEG files ----------------------------------------------------
 * The last stage of a device pipeline: the coefficients decode_async / run_async leave on the GPU
 * written as the sequential Huffman JPEG file the jpegqs tool writes for them (its writer, jpegcoef.c
 * jq_write), byte for byte.
 *
 * The prefix: what jq_write puts before its first DQT - SOI, the JFIF APP0 (grayscale / YCbCr, with
 * the input's version and density) or Adobe APP14 (RGB / CMYK / YCCK), then the input's APPn / COM
 * markers copied at level `copy` (0 none, 1 COM, 2 COM + APPn; the tool's -c), markers between the
 * scans of a progressive file included.  It depends on the input file only.  Host-only: walks the
 * file's markers without decoding entropy-coded data.  *out_len receives the prefix length (out may
 * be NULL to ask for it), *ncomp the frame's component count, comp_id / quant_tbl its component
 * identifiers and quantization table numbers (entries past the component count 0).  Returns 0, or JPEGQS_ERR_ARG for what the
 * tool's reader rejects or when the prefix does not fit cap (jpegqs_cuda_last_error(NULL)). */
int jpegqs_cuda_jpeg_prefix(const uint8_t *data, size_t len, int copy, uint8_t *out, size_t cap, size_t *out_len,
		int32_t *ncomp, int32_t comp_id[4], int32_t quant_tbl[4]);

/* What the device writes in front of the entropy-coded data of image i besides the DQT, SOF, DHT and
 * SOS segments: jpegqs_cuda_jpeg_prefix's output, in DEVICE memory, and the frame's identifiers. */
typedef struct {
	const uint8_t *prefix_dev;   /* DEVICE memory: the prefix bytes (host memory for encode_model) */
	uint32_t prefix_len;
	int32_t comp_id[4];          /* SOF / SOS component identifiers                                */
	int32_t quant_tbl[4];        /* SOF quantization table numbers (0..3); DQT follows them        */
} jpegqs_cuda_jpeg_head;

/* Stream-ordered, graph-capturable encode of n images' coefficients to JPEG files on the GPU.
 *   - What it writes.  For image i: heads[i]'s prefix, then what jq_write(..., optimize) writes for
 *     these coefficients, geometry and quant tables: DQT for each table in use in component order
 *     (16-bit, with SOF1, when a value exceeds 255), SOF0 / SOF1, DHT - with optimize 0 the T.81 K.3.3
 *     tables, with optimize 1 optimal tables built from this image's symbol counts (T.81 K.2 with
 *     jq_write's tie-breaking), two table pairs when there is more than one component - SOS, one
 *     interleaved sequential scan without restart markers, EOI.  Blocks of the MCU padding code a DC
 *     difference of 0 and no AC (libjpeg's jctrans.c), the last byte is filled with 1-bits, 0xFF
 *     bytes are stuffed.  quant[] of a component with has_qtbl is written as its table (the values,
 *     ones after run_async, are not applied to the coefficients).
 *   - Inputs.  comp[].coef / coef_up: DEVICE pointers on the context's device, 16-byte aligned, of
 *     libjpeg's wblk / hblk; rows / rows_up NULL.  1-4 components, sampling factors 1..4, at most 10
 *     blocks per MCU, image size 1..65535.
 *   - Chroma source, render_async's rule.  An image UPSAMPLE_UV can up-sample (YCbCr, three components,
 *     chroma 1x1, luma not) is written "up-sampled" - components 1 and 2 from coef_up, all three
 *     sampled 1x1 at the luma's block geometry, what do_quantsmooth leaves in cinfo - when
 *       . run_status_dev != NULL: run_status_dev[i].upsampled != 0 on the device, for images whose two
 *         coef_up pointers are set.  So one graph may hold decode -> run_async -> encode, and a replay
 *         in which an image stops writes it at its sampling.  An image that can be up-sampled but was
 *         given no coef_up is written as sampled; if the run status says it was up-sampled, its status
 *         gets JPEGQS_ENCODE_NO_UP (the file is valid, but its chroma is not what the tool writes).
 *       . run_status_dev == NULL: imgs[i].upsampled != 0 (coef_up then required).
 *   - Output.  out_dev[i]: out_cap[i] bytes of device memory at any alignment.  len_dev[i] (device
 *     uint64) receives the file length, status_dev[i] (device int32) 0 or an OR of the bits below.
 *     On OVERFLOW len_dev[i] holds the length the file needs and nothing is written at or past
 *     out_cap[i].  On RANGE the file is not valid (jq_write fails there with "coefficient out of range
 *     for Huffman coding"); the writes stay inside out_cap[i] all the same.  A flagged image does not
 *     affect the others.
 *   - Bound.  jpegqs_cuda_encode_bound returns a capacity that never overflows: with U the blocks of
 *     the scan (MCUs x blocks per MCU; the larger of the two geometries for an image that can be
 *     up-sampled), prefix_len + 1680 + 2 * ceil(U * 1665 / 8) - a block codes to at most 1665 bits,
 *     stuffing at most doubles the bytes, and DQT + SOF + DHT + SOS + EOI take at most 1680.
 *   - Argument errors change nothing: every check runs before the first enqueue and a failed one
 *     returns JPEGQS_ERR_ARG with nothing enqueued.  Checked: NULL pointers (imgs, heads, out_dev and
 *     its entries, out_cap, len_dev, status_dev, workspace, coef, a prefix_dev of a non-empty prefix),
 *     rows / rows_up set, coef / coef_up not 16-byte aligned, ncomp outside 1..4, sampling factors
 *     outside 1..4, more than 10 blocks per MCU, wblk / hblk other than libjpeg's, an image size
 *     outside 1..65535, comp_id outside 0..255 or quant_tbl outside 0..3, imgs[i].upsampled on an
 *     image that cannot be up-sampled or without coef_up (run_status_dev NULL), a workspace too small
 *     or not 256-byte aligned, and out_cap[i] < prefix_len.  A CUDA error while enqueueing returns
 *     JPEGQS_ERR_CUDA.
 *   - The stream rules of decode_async: no cudaMalloc, no synchronisation, no event record or query.
 *     Descriptors, quant tables and the standard Huffman tables travel as kernel parameters; nothing
 *     of imgs or heads is read after return.  Legal under cudaStreamCaptureModeGlobal: a replay
 *     encodes the current contents of the same coefficient, prefix and status buffers with the
 *     geometry, quant tables and identifiers fixed at capture.  Two calls on different streams with
 *     separate workspaces may be in flight together.  jpegqs_cuda_last_launches counts the launches
 *     (nine per group of up to 16 images, ten with optimize); larger batches run as several groups,
 *     one after another on the stream.
 *   - Workspace: all per-call device state.  With A(x) = x rounded up to a multiple of 256 and U as
 *     for the bound, T = ceil(U / 256), W = ceil(U * 1665 / 32) + 2, the size is the sum over images of
 *       32768 + A(2 * U) + A(8 * T) + A(4 * W) + A(4 * ceil(4 * W / 4096))
 *     (descriptor, state and tables; bits per block; bits per tile; the unstuffed bits, sized for the
 *     worst case; 0xFF counts per 4 KB).  It does not depend on optimize.  An 8K (7680 x 4320) 4:2:0
 *     image that can be up-sampled has U = 1 555 200 and needs 324 MB, most of it the bit buffer.
 * Returns 0 or a negative error. */
#define JPEGQS_ENCODE_RANGE    1   /* a DC difference of category > 11 or an AC value of category > 10 */
#define JPEGQS_ENCODE_OVERFLOW 2   /* the file does not fit out_cap; len_dev holds the size it needs   */
#define JPEGQS_ENCODE_NO_UP    4   /* run status up-sampled, coef_up not given: written as sampled     */
int jpegqs_cuda_encode_bound(const jpegqs_cuda_image *img, size_t prefix_len, size_t *bytes);
int jpegqs_cuda_encode_workspace_bytes(int n, const jpegqs_cuda_image *imgs, int optimize, size_t *bytes);
int jpegqs_cuda_encode_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_jpeg_head *heads, int optimize, const jpegqs_cuda_status *run_status_dev,
		uint8_t *const *out_dev, const size_t *out_cap, uint64_t *len_dev, int32_t *status_dev,
		void *workspace, size_t workspace_bytes, void *stream);
/* jpegqs_cuda_encode_async's algorithm on the CPU for one image: the same unit, predictor, table,
 * header and stuffing functions in the same order on one thread.  img->comp[c].coef / coef_up and
 * head->prefix_dev are HOST memory; imgs->upsampled picks the geometry.  *len / *status as len_dev /
 * status_dev.  Returns 0 or JPEGQS_ERR_ARG. */
int jpegqs_cuda_encode_model(const jpegqs_cuda_image *img, const jpegqs_cuda_jpeg_head *head, int optimize,
		uint8_t *out, size_t cap, uint64_t *len, int32_t *status);

/* ---- JPEG file -> smoothed JPEG file, blocking --------------------------------------------------
 * The jpegqs tool's transcode (read, do_quantsmooth, write) on the device: decode, smoothing and
 * encode kernels on one stream, only the file's bytes crossing the bus.
 *
 * The route.  Host-only, no device needed, safe to call from any thread (it writes no error state).
 * A file goes to the DEVICE only when all of these hold, else to the HOST (the tool's reader,
 * do_quantsmooth and writer):
 *   - the markers-only walk of the whole file meets no error and none of the reader's marker-level
 *     warnings (bytes before a marker, no EOI), so the tool would exit 0 on it;
 *   - jpegqs_cuda_jpeg_parse takes it (and it has one scan), or jpegqs_cuda_jpeg_parse_scans does;
 *   - it is not a progressive file with an AC refinement scan without restart markers: the device
 *     decodes such a scan on one thread, about 13x slower than the host reader (DESIGN.md 3.6.1);
 *   - it has at most 4 components and, with several, at most 10 blocks per MCU (the encoder's limits).
 * Returns JPEGQS_ROUTE_DEVICE, JPEGQS_ROUTE_HOST or JPEGQS_ERR_ARG (the reader rejects the file).
 * *reason (may be NULL) receives a short static description for traces.  info (may be NULL) receives
 * what the tool's -v line shows. */
#define JPEGQS_ROUTE_HOST   0
#define JPEGQS_ROUTE_DEVICE 1
typedef struct {
	uint32_t image_width, image_height;
	int32_t ncomp, progressive;
	int32_t restart_interval;          /* the last DRI of the file, as the reader reports it */
} jpegqs_cuda_file_info;
int jpegqs_cuda_transcode_route(const uint8_t *data, size_t len, const char **reason, jpegqs_cuda_file_info *info);

/* The transcode.  data / len: a JPEG file in host memory.  flags, niter: do_quantsmooth's (flags &
 * JPEGQS_FLAGS_MASK is used); optimize, copy: the tool's -o and -c.  The call routes the file itself,
 * uploads it through pinned staging, runs decode_async (one sequential scan) or decode_scans_async,
 * then run_async - unless do_quantsmooth would return early without touching the coefficients (niter
 * <= 0 and UPSAMPLE_UV with nothing to up-sample) - then encode_async with the run status and the
 * up-sampled chroma, so up-sampled and stopped images are written as the tool writes them, and waits.
 * Returns
 *   JPEGQS_TRANSCODE_OK        result->data / len hold the file the tool writes, byte for byte;
 *   JPEGQS_TRANSCODE_FALLBACK  the host route must take this file: the route says HOST, the device
 *                              decoder flagged the data (any JPEGQS_DECODE_* bit) or the encoder met
 *                              a coefficient it cannot code (JPEGQS_ENCODE_RANGE).  The host route
 *                              gives the reader's recovery, warning count and messages.
 *                              result->reason says which;
 *   < 0                        JPEGQS_ERR_ARG (arguments, a file the reader rejects) or
 *                              JPEGQS_ERR_CUDA (jpegqs_cuda_last_error(ctx)).
 * Output memory: result->data is allocated by the library with malloc(); release it with
 * jpegqs_cuda_transcode_free (which is free()).  Device memory: the file, the coefficients, the
 * up-sampled chroma, one workspace shared by the three stages (they run one after another on the
 * stream) and the output belong to the context, only grow, and are kept between calls, so a run of
 * files of similar sizes makes no cudaMalloc / cudaFree.  jpegqs_cuda_last_device_ms gives the
 * smoothing kernels' time (CUDA events around run_async).  One calling thread per context, like the
 * other blocking entry points. */
#define JPEGQS_TRANSCODE_OK       0
#define JPEGQS_TRANSCODE_FALLBACK 1
typedef struct {
	uint8_t *data; size_t len;         /* OK: the output file (malloc'd)                              */
	int32_t smoothed;                  /* 1 = run_async ran (0: do_quantsmooth's early return)        */
	int32_t stop, upsampled;           /* the run's status when it ran (0 when the decoder flagged the
	                                      data: the run then went over unspecified coefficients)      */
	const char *reason;                /* FALLBACK: why, a static string; "" otherwise                */
} jpegqs_cuda_transcode_result;
int jpegqs_cuda_transcode(jpegqs_cuda_ctx *ctx, const uint8_t *data, size_t len, int flags, int niter,
		int optimize, int copy, jpegqs_cuda_transcode_result *result);
void jpegqs_cuda_transcode_free(void *p);

/* The transcode of n files in shared launches (jpegqs_cuda_transcode is the batch of one).
 *   - Per file.  rc[i] and results[i] are exactly what jpegqs_cuda_transcode returns for file i alone:
 *     JPEGQS_TRANSCODE_OK, JPEGQS_TRANSCODE_FALLBACK or JPEGQS_ERR_ARG for a file the reader rejects
 *     (jpegqs_cuda_last_error(ctx) names the last such file), with the same bytes, smoothed, stop,
 *     upsampled and reason.  A file that falls back or stops never changes another file's result.
 *   - Return.  0, or a negative error for bad arguments (ctx, data, len, rc or results NULL, a data[i]
 *     NULL, n < 0, copy outside 0..2: nothing is done) or a CUDA failure.  On a negative return every
 *     results[i].data is NULL.  n == 0 returns 0 and touches nothing.
 *   - Sub-batches.  Consecutive device-route files are grouped while the sum of their needs stays
 *     within max_device_bytes: file + prefix, coefficients (+ up-sampled chroma), the encoder's bound
 *     for the output, and one workspace shared by the stages - the largest of the decoders', run_async's
 *     and the encoder's workspace for the group and of the packed output (the bounds again, each
 *     rounded up to 16 bytes).  A file bigger than the budget runs alone; at most 1024 files go in one
 *     sub-batch.  max_device_bytes 0: half of the device memory free at call time plus what the
 *     context's transcode buffers already hold.  The buffers belong to the context and only grow.
 *   - Per sub-batch, on the context's stream: one upload of all files and prefixes from pinned
 *     staging; one decode_async over the single-scan files and one decode_scans_async over the others;
 *     one run_async over the files that smooth (do_quantsmooth's early return is decided per file, and
 *     the files that return early get run status 0); one encode_async over all; one packing kernel
 *     that copies the clean files into one buffer; the status records back, a synchronisation, exactly
 *     the packed bytes back, a synchronisation.
 *   - jpegqs_cuda_last_device_ms gives the run_async time of the last sub-batch that smoothed. */
int jpegqs_cuda_transcode_batch(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int optimize, int copy, size_t max_device_bytes, int *rc,
		jpegqs_cuda_transcode_result *results);

/* ---- JPEG files -> smoothed pixels, blocking, many files per launch -----------------------------
 * What the jpegqs tool's --ppm writes after its P5 / P6 header, for n files in host memory: libjpeg's
 * islow, fancy-up-sampled pixels of the coefficients do_quantsmooth(flags, niter) leaves, so
 * up-sampled and stopped images come out as the tool renders them.
 *   - Output size.  out[i] holds exactly image_width * image_height * channels bytes, where width,
 *     height and ncomp are what jpegqs_cuda_transcode_route puts in its info for file i and channels
 *     is 1 for ncomp 1 (grey) and 3 for ncomp 3 (RGB).  layout JPEGQS_RENDER_HWC or _CHW (the same
 *     bytes for a grey file).  out_on_device 1: out[i] is device memory on the context's device, at
 *     any byte alignment; 0: host memory, filled from one download per sub-batch.  Either way the
 *     call blocks and the outputs are complete when it returns.
 *   - Per file, rc[i]: 0; JPEGQS_ERR_ARG for a file the reader rejects (jpegqs_cuda_last_error(ctx)
 *     names the last such file); JPEGQS_ERR_UNSUPPORTED for a component count other than 1 or 3 or a
 *     sampling render_async does not render (--ppm fails on these with "render failed (-3)").  out[i]
 *     is then untouched.  A file that fails never changes another file's result.
 *   - Route.  jpegqs_cuda_transcode_route's, unchanged.  DEVICE files are uploaded and decoded by
 *     decode_async / decode_scans_async in shared launches; HOST files are read by
 *     jpegqs_cuda_jpeg_read into pinned staging, on the calling thread while the device decodes; a
 *     DEVICE file the device decoder flags is read again by jpegqs_cuda_jpeg_read, as the tool does
 *     when a transcode falls back, so its warnings and recovery are the reader's.
 *   - Per sub-batch, on the context's stream: one upload of the DEVICE files; the decoder launches;
 *     the host reads; the decoder statuses back and a synchronisation; the re-reads; one upload of
 *     the host-decoded coefficients; one run_async over the files that smooth (do_quantsmooth's early
 *     return decided per file, as in transcode_batch); one render of every file, reading the run
 *     status and the up-sampled chroma; the run statuses back (with the pixels when out_on_device is
 *     0) and a synchronisation.
 *   - Sub-batches, as transcode_batch's: consecutive files while the sum of their needs stays within
 *     max_device_bytes (0: half of the free device memory plus what the context's buffers hold), at
 *     most 1024 files, a bigger file alone.  The needs: the file, the coefficients and up-sampled
 *     chroma, the shared workspace (the decoders' and run_async's) and, with host outputs, the
 *     pixels.  A re-read file takes its coefficient bytes once more.  The buffers belong to the
 *     context and only grow.  jpegqs_cuda_last_device_ms gives the run_async time of the last
 *     sub-batch that smoothed.
 *   - Return.  0, or a negative error for bad arguments (ctx, data, len, out, rc or results NULL, an
 *     entry of data or out NULL, n < 0, a layout other than HWC / CHW, out_on_device other than 0 / 1:
 *     nothing is done and rc / results are untouched) or a CUDA failure.  n == 0 returns 0. */
typedef struct {
	int32_t channels;        /* 1 (grey) or 3 (RGB)                                               */
	int32_t host_decoded;    /* 1: the host reader decoded the entropy-coded data                  */
	int32_t warnings;        /* the host reader's warning count (the tool would exit 2 if > 0)     */
	int32_t smoothed, stop, upsampled;   /* as jpegqs_cuda_transcode_result                       */
	const char *reason;      /* host_decoded: why (a static string), "" otherwise                  */
} jpegqs_cuda_pixels_result;
int jpegqs_cuda_pixels_batch(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int out_on_device, uint8_t *const *out, size_t max_device_bytes,
		int *rc, jpegqs_cuda_pixels_result *results);

/* The same files at 1/2, 1/4 or 1/8 size (jpegqs_cuda_pixels_batch is this call with scale_denom 1):
 * the routes, sub-batches, warnings, host_decoded, smoothed, stop and upsampled are those of the
 * unscaled call, and only the render differs - jpegqs_cuda_render_scaled_async's.
 *   - Output size.  out[i] holds exactly ceil(width / d) * ceil(height / d) * channels bytes, d =
 *     scale_denom, with width, height and channels as for jpegqs_cuda_pixels_batch.  A 1920 x 1080
 *     colour file at d = 4 gives 480 x 270 x 3 bytes.  With host outputs each file's share of the
 *     sub-batch budget and of the download is its scaled size.
 *   - Pixels.  Byte for byte what libjpeg's jpeg_read_scanlines gives with scale_num 1, scale_denom d,
 *     JDCT_ISLOW and fancy up-sampling, JCS_RGB (JCS_GRAYSCALE for a grey file), for the coefficients
 *     the render reads at d = 1: for a file that smooths, those of the file jpegqs writes for the same
 *     flags and niter; for a file do_quantsmooth returns early on, those of the input file.
 *   - Return.  As jpegqs_cuda_pixels_batch's, and a scale_denom outside {1, 2, 4, 8} is a bad argument
 *     (JPEGQS_ERR_ARG, nothing done). */
int jpegqs_cuda_pixels_batch_scaled(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int out_on_device, uint8_t *const *out,
		size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results);

/* ---- the same files cropped and resized: Pillow's Image.resize, byte for byte --------------------
 * File i's output is exactly what Pillow gives for
 *     Image.fromarray(P).crop((left, top, right, bottom)).resize((width, height), filter)
 * where P is what jpegqs_cuda_pixels_batch_scaled gives for the file at the same scale_denom, as an
 * 'RGB' picture, or 'L' for a grey file.  The filters are Pillow's convolution filters, numbered as
 * its Image.Resampling; NEAREST (0) takes another code path in Pillow and is rejected.
 *   - Output size.  out[i] holds exactly width * height * channels bytes in layout HWC or CHW, with
 *     channels as for jpegqs_cuda_pixels_batch.  With host outputs each file's share of the budget and
 *     of the download is its resized size.
 *   - Everything else - routes, sub-batches, warnings, host_decoded, smoothed, stop, upsampled - is
 *     pixels_batch_scaled's for the same files.
 *   - Arithmetic.  Pillow's (Resample.c): per axis, weights computed in double on the host and rounded
 *     to int32 with 22 fractional bits; a horizontal pass over the rows the vertical pass reads, into
 *     an 8-bit intermediate, then the vertical pass; each output byte is clip8(2^21 + sum src * k).
 *   - Per sub-batch: the render writes each file's 1/scale_denom picture (HWC) to a context buffer;
 *     one upload carries the resize descriptors and weight tables; two launches over all the files
 *     write the outputs.  The budget counts the picture, the intermediate and the tables of each file,
 *     and with host outputs the resized bytes.
 *   - Per file, rc[i]: as pixels_batch_scaled's, and JPEGQS_ERR_ARG for a crop outside the file's
 *     1/scale_denom picture, or an empty one (jpegqs_cuda_last_error(ctx) names the file); out[i] is
 *     then untouched and no other file changes.
 *   - Return.  As pixels_batch_scaled's; also JPEGQS_ERR_ARG with nothing done for boxes NULL, a
 *     filter other than the five below, or a width or height outside 1..65535. */
#define JPEGQS_RESIZE_LANCZOS  1   /* Pillow's Image.Resampling values */
#define JPEGQS_RESIZE_BILINEAR 2
#define JPEGQS_RESIZE_BICUBIC  3
#define JPEGQS_RESIZE_BOX      4
#define JPEGQS_RESIZE_HAMMING  5
typedef struct {
	int32_t left, top, right, bottom;  /* crop in the 1/scale_denom picture; all 0: the whole picture */
	int32_t width, height;             /* output size */
} jpegqs_cuda_resize_box;
int jpegqs_cuda_pixels_batch_resized(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results);

/* The resize of jpegqs_cuda_pixels_batch_resized on the calling thread, for one picture (host-only, no
 * device needed): the same weight tables and per-pixel arithmetic.  src: width x height x channels
 * bytes, HWC; channels 1 or 3.  out: box->width * box->height * channels bytes in layout HWC or CHW.
 * Returns 0, or JPEGQS_ERR_ARG (NULL pointer, bad size, channels, layout or filter, a crop outside
 * the picture or empty); jpegqs_cuda_last_error(NULL) says why. */
int jpegqs_cuda_resize_model(const uint8_t *src, int width, int height, int channels, int layout, int filter,
		const jpegqs_cuda_resize_box *box, uint8_t *out);

/* jpegqs_cuda_pixels_batch_resized (boxes != NULL) or _scaled (boxes NULL, filter ignored) with one
 * orientation per file: 1..8 as for jpegqs_cuda_render_oriented_async, or JPEGQS_ORIENT_FILE (0) for
 * the file's own (jpegqs_cuda_jpeg_orientation's).  orientation NULL is 1 for every file: the call is
 * then byte for byte the existing one.
 *   - The render writes the oriented picture; the crop and the resize then take it as it is, so a box
 *     is in the oriented 1/d picture (Pillow's exif_transpose, then crop, then resize).  A crop valid
 *     only in the unoriented picture fails that file alone with JPEGQS_ERR_ARG.
 *   - Unresized, out[i] is the oriented picture: for 5..8, H' x W' x C (or C planes of H' rows of W')
 *     with W' and H' as in the table above - the same number of bytes.  Budgets do not change.
 *   - Return.  As the existing calls', and an entry outside 0..8 is a bad argument (JPEGQS_ERR_ARG,
 *     nothing done). */
int jpegqs_cuda_pixels_batch_oriented(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const int32_t *orientation, int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results);

/* jpegqs_cuda_pixels_batch_oriented with a colour mode (JPEGQS_PIXELS_*; 0 is byte for byte the oriented
 * call).  With mode RGB or L:
 *   - channels, out[i]'s size, results[i].channels, the budgets and the crop and resize are those of a
 *     3-channel (RGB) or 1-channel (L) picture for every file; CHW and HWC are the same bytes for L.
 *   - 4-component files (CMYK, YCCK) are rendered - their colour space is the header's - and smoothed as
 *     the tool smooths them; sampling ratios that are not integral are JPEGQS_ERR_UNSUPPORTED per file.
 *   - file i gives Pillow's im = Image.open(F) (im.draft(None, (W // d, H // d)) at d > 1), then
 *     exif_transpose or the explicit transpose, then im.convert(mode), then crop and resize, with F the
 *     file jpegqs writes for the same flags and niter (the input where do_quantsmooth returns early).
 *   - A mode other than 0, 1, 2 is a bad argument (JPEGQS_ERR_ARG, nothing done). */
int jpegqs_cuda_pixels_batch_mode(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const int32_t *orientation, int mode, int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results);

/* ---- 8-bit pictures -> JPEG files: Pillow's Image.save, byte for byte ---------------------------
 * Picture i's file is exactly what Pillow (with its libjpeg-turbo) writes for
 *     Image.fromarray(P).save(f, "JPEG", quality=quality, subsampling=subsampling, optimize=optimize)
 * where P is the picture as an 'RGB' (channels 3) or 'L' (channels 1) image.  That is plain libjpeg:
 * jpeg_set_defaults, jpeg_set_quality(quality, force_baseline TRUE), luma sampling 1x1 / 2x1 / 2x2 for
 * subsampling 0 / 1 / 2 (4:4:4, 4:2:2, 4:2:0, Pillow's numbering; grey pictures ignore it), chroma 1x1,
 * optimize_coding = optimize, islow DCT, component ids 1, 2, 3, quantization table 0 for luma and 1 for
 * both chroma components, and the JFIF 1.01 APP0 with density unit 0 and density 1:1.
 *   - The compressor kernel restates jccolor.c's rgb_ycc_convert (16-bit fixed point), jcsample.c's
 *     fullsize / h2v1 / h2v2 down-sampling (alternating biases 0,1 and 1,2), jcprepct.c's edges (the
 *     right edge repeats the last full-resolution column before down-sampling; the bottom edge repeats
 *     the last down-sampled row), jfdctint.c's jpeg_fdct_islow on sample - 128 and jcdctmgr.c's
 *     quantization (sign(t) * ((|t| + 4q) / (8q))).  Geometry is libjpeg's: downsampled width =
 *     ceil(W * h / max_h), width in blocks = ceil(downsampled width / 8), and the same for heights.
 *   - jpegqs_cuda_encode_async then writes the coefficients, so the files are its output for them.
 *   - Grey pictures: the samples do not depend on subsampling, but Pillow sets the luma sampling factors
 *     whatever the component count, so the SOF of a grey file saved with 4:2:2 / 4:2:0 says 2x1 / 2x2
 *     (its single-component scan is coded block by block all the same); so does this one.
 *   - Progressive files: optimize | JPEGQS_JPEG_PROGRESSIVE gives Pillow's save(..., progressive=True),
 *     libjpeg's jpeg_simple_progression with optimal tables, which progressive mode forces: bit 0 then
 *     changes no byte.  SOF2, then per scan the DHT of every table the scan uses (one marker each,
 *     tables built from that scan's symbol counts; none for the DC refinement), SOS and the scan's data,
 *     padded with 1-bits and byte-stuffed on its own.  The scans (Ss-Se, Ah, Al):
 *       YCbCr  DC of all three 0-0 0 1; Y 1-5 0 2; Cr 1-63 0 1; Cb 1-63 0 1; Y 6-63 0 2; Y 1-63 2 1;
 *              DC 0-0 1 0; Cr 1-63 1 0; Cb 1-63 1 0; Y 1-63 1 0.
 *       grey   DC 0-0 0 1; 1-5 0 2; 6-63 0 2; 1-63 2 1; DC 0-0 1 0; 1-63 1 0.
 *     Any other optimize value (2, 4, 0x200, ...) is JPEGQS_ERR_ARG.  Callers that never set the bit
 *     get the sequential files and sizes described here. */
#define JPEGQS_JPEG_PROGRESSIVE 0x100
typedef struct {
	int32_t quality;       /* 1..100                                                               */
	int32_t subsampling;   /* 0 = 4:4:4, 1 = 4:2:2, 2 = 4:2:0 (Pillow's numbers); ignored for grey   */
	int32_t optimize;      /* 0 / 1: optimal Huffman tables; | JPEGQS_JPEG_PROGRESSIVE: progressive   */
} jpegqs_cuda_jpeg_params;
typedef struct {
	const uint8_t *pixels_dev; /* DEVICE memory (host memory for compress_model), HWC, any alignment  */
	int32_t width, height;     /* 1..65535                                                         */
	int32_t channels;          /* 1 (grey) or 3 (RGB)                                              */
	size_t row_bytes;          /* bytes from one row to the next, >= width * channels              */
} jpegqs_cuda_pixels_in;

/* Stream-ordered, graph-capturable compression of n device pictures with one params for all.
 *   - Per group of up to 32 pictures, one compressor launch turns every component into quantized
 *     coefficients in the workspace; then jpegqs_cuda_encode_async writes them with the scaled tables
 *     and the JFIF prefix (the compressor kernel copies the prefix from its parameters into the
 *     workspace).  jpegqs_cuda_last_launches counts both.
 *   - Output.  out_dev[i]: out_cap[i] bytes of device memory at any alignment; len_dev[i] (device
 *     uint64) and status_dev[i] (device int32) as encode_async's: 0, or JPEGQS_ENCODE_OVERFLOW with
 *     len_dev[i] the length the file needs and nothing written at or past out_cap[i].  RANGE cannot
 *     occur for 8-bit samples.
 *   - Bound.  jpegqs_cuda_compress_bound: encode_bound with a 20-byte prefix, 20 + 1680 +
 *     2 * ceil(U * 1665 / 8), with U = MCUs x blocks per MCU: ceil(W/8) * ceil(H/8) for grey,
 *     3 * ceil(W/8) * ceil(H/8) for 4:4:4, 4 * ceil(W/16) * ceil(H/8) for 4:2:2 and
 *     6 * ceil(W/16) * ceil(H/16) for 4:2:0.
 *   - Workspace.  With A(x) = x rounded up to a multiple of 256, jpegqs_cuda_compress_workspace_bytes is
 *     256 (the prefix) plus, per picture, sum over components of A(128 * wblk * hblk) (the
 *     coefficients) plus encode_workspace_bytes' term for the picture's geometry:
 *       32768 + A(2 * U) + A(8 * T) + A(4 * Wd) + A(4 * ceil(4 * Wd / 4096)),
 *     T = ceil(U / 256), Wd = ceil(U * 1665 / 32) + 2.  The workspace is 256-byte aligned.
 *   - Progressive bound and workspace (JPEGQS_JPEG_PROGRESSIVE set): 20 + 6000 + 2 * (ceil(U * 3928 / 8)
 *     + 10), with 3928 a block's bits over all scans at most (DESIGN.md 3.14); U below 2^27 for 65535 x
 *     65535, so no term overflows 64 bits.  The encoder's term becomes
 *       73728 + A(V) + A(2 * V) + A(8 * V) + A(2 * V) + A(8 * V / 256) + A(4 * Wd) + A(4 * ceil(4 * Wd / 4096)),
 *     Wd = ceil(U * 3928 / 32) + 10242, V = the sum over the scans of their units rounded up to a
 *     multiple of 256: R(U) twice (the DC scans), R(Y) four times and R(C) twice for each chroma
 *     component, Y and C = wblk * hblk of the component (grey: R(U) six times).
 *   - Launches: the compressor, then 13 per group of up to 16 pictures in progressive mode (9 / 10 in
 *     sequential mode), then the grey SOF fix where it applies.
 *   - Argument errors change nothing: every check runs before the first enqueue and a failed one
 *     returns JPEGQS_ERR_ARG with nothing enqueued.  Checked: NULL pointers (pics, params, out_dev and
 *     its entries, out_cap, len_dev, status_dev, workspace, pixels_dev), quality outside 1..100,
 *     subsampling outside 0..2, optimize other than 0 / 1, width or height outside 1..65535, channels
 *     other than 1 or 3, row_bytes < width * channels, out_cap[i] < 20, a workspace too small or not
 *     256-byte aligned.
 *   - encode_async's stream rules: no cudaMalloc, no synchronisation; descriptors, tables and the
 *     prefix travel as kernel parameters and nothing of pics or params is read after return.  A
 *     replay of a captured call compresses the current contents of the same pixel buffers. */
int jpegqs_cuda_compress_bound(const jpegqs_cuda_pixels_in *pic, const jpegqs_cuda_jpeg_params *params, size_t *bytes);
int jpegqs_cuda_compress_workspace_bytes(int n, const jpegqs_cuda_pixels_in *pics, const jpegqs_cuda_jpeg_params *params,
		size_t *bytes);
int jpegqs_cuda_compress_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_pixels_in *pics,
		const jpegqs_cuda_jpeg_params *params, uint8_t *const *out_dev, const size_t *out_cap, uint64_t *len_dev,
		int32_t *status_dev, void *workspace, size_t workspace_bytes, void *stream);
/* The same per-block functions and encode_model on the calling thread, for one picture whose pixels_dev
 * is HOST memory (no device needed).  *len / *status as len_dev / status_dev.  Returns 0 or
 * JPEGQS_ERR_ARG (the checks of compress_async; cap < 20); jpegqs_cuda_last_error(NULL) says why. */
int jpegqs_cuda_compress_model(const jpegqs_cuda_pixels_in *pic, const jpegqs_cuda_jpeg_params *params,
		uint8_t *out, size_t cap, uint64_t *len, int32_t *status);

/* JPEG files in, JPEG files out: each file's picture as jpegqs_cuda_pixels_batch_resized gives it (boxes
 * given) or jpegqs_cuda_pixels_batch_scaled (boxes NULL), written as Pillow's Image.save(quality,
 * subsampling, optimize) writes it (compress_async's files).  A grey file gives a grey JPEG.
 *   - Per sub-batch, after the render (and resize) into the context's buffers: compress_async over the
 *     pictures, then the packing kernel of transcode_batch; only the packed files and the statuses
 *     come back.
 *   - out[i] receives a malloc'd file of out_len[i] bytes (release it with jpegqs_cuda_transcode_free),
 *     or NULL for a file that fails.  rc[i], routes, warnings and results[i] are those of the pixel
 *     call for the same files; a bad file or a bad crop fails alone.
 *   - The budget counts, per file, what the pixel call counts with host outputs, plus the compressor's
 *     workspace share (coefficients and encoder workspace) and the bound, twice (slot and packed copy).
 *   - Return.  As pixels_batch_resized's (0, or a negative error with nothing done for bad arguments:
 *     also params NULL or out of range, out_len NULL); on a negative return every out[i] is NULL. */
int jpegqs_cuda_pixels_batch_jpeg(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len);

/* jpegqs_cuda_pixels_batch_jpeg with orientation as for jpegqs_cuda_pixels_batch_oriented: file i is
 * Pillow's exif_transpose(P) (or P.transpose for an explicit value), then crop / resize, then save - a
 * JFIF file with upright pixels and no orientation tag.  NULL: byte for byte pixels_batch_jpeg. */
int jpegqs_cuda_pixels_batch_jpeg_oriented(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len, const int32_t *orientation);

/* jpegqs_cuda_pixels_batch_jpeg_oriented with a colour mode as for jpegqs_cuda_pixels_batch_mode: the
 * converted picture is saved (an L picture as a grey file).  Mode 0: byte for byte the oriented call. */
int jpegqs_cuda_pixels_batch_jpeg_mode(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len, const int32_t *orientation, int mode);

/* ---- thumbnails and reducing_gap: Pillow's Image.thumbnail and Image.resize(reducing_gap=) --------
 * Pillow's thumbnail((bw, bh), filter, reducing_gap) of a W x H JPEG file:
 *   1. the size: preserve_aspect_ratio (round_aspect of the bound's aspect), or nothing at all when the
 *      bound covers the picture on both axes;
 *   2. the draft scale s: the first of 8, 4, 2, 1 at most min(W // int(bw * gap), H // int(bh * gap)),
 *      and the picture at 1/s (libjpeg's scaled decode); no draft for gap None, or when the picture was
 *      loaded first (exif_transpose, transpose and convert load it, and draft then does nothing);
 *   3. no resize when the drafted picture already has the thumbnail's size; otherwise
 *      Image.resize(size, filter, box = (0, 0, W / s, H / s), reducing_gap):
 *   4. factor = int(box_w / out_w / gap) or 1 per axis; when one is above 1, Image.reduce by the factors
 *      over _get_safe_box (the box widened by the filter's support less 0.5 in source samples, then
 *      rounded outwards), and the box shifted and divided by the factors;
 *   5. the convolution resize of the (reduced) picture from that box, which Pillow's C layer takes as
 *      float: scale = (double)(float)(in1 - in0) / out, centres in0 + (xx + 0.5) * scale in double.
 * Reduce arithmetic (Reduce.c): each output sample covers the n = fx * fy samples of its cell, fewer in
 * the partial cells at the right and bottom edges of the box, and is ((sum + n / 2) * m) >> 24 with
 * m = (uint32)((float)2^32 / (float)(256 * n)), in 32-bit unsigned arithmetic - not the rounded mean.
 * A cell of 2^23 samples or more (256 * n would overflow Pillow's int) is refused; so is a picture more
 * than 100 times taller than wide after the reduce, which Pillow resizes vertically first.  Both fail the
 * file alone with JPEGQS_ERR_ARG.
 *
 * jpegqs_cuda_thumbnail_geometry: steps 1 and 2 (host-only), so callers can size out[i].  width and
 * height are the picture thumbnail sees (oriented for 5..8); loaded = 1 when an orientation or a mode is
 * given (then *scale_denom is 1).  reducing_gap 0.0 means None, otherwise finite and at least 1.0; bounds
 * and sizes 1..65535.  Returns 0 or JPEGQS_ERR_ARG; jpegqs_cuda_last_error(NULL) says why. */
int jpegqs_cuda_thumbnail_geometry(int width, int height, int bound_w, int bound_h, double reducing_gap, int loaded,
		int *scale_denom, int *out_w, int *out_h);

/* jpegqs_cuda_pixels_batch_mode with thumbnails and reducing_gap.  reducing_gap 0.0 means None; any
 * other value must be finite and at least 1.0.
 *   - thumbnail 0: boxes mean what they mean for the mode call, and file i is Pillow's
 *     Image.fromarray(P).crop(box).resize(size, filter, reducing_gap=reducing_gap); reducing_gap 0.0 is
 *     byte for byte the mode call.
 *   - thumbnail 1: file i is Pillow's Image.open(F) [exif_transpose / transpose] [convert(mode)] then
 *     thumbnail((boxes[i].width, boxes[i].height), filter, reducing_gap) (steps 1-5 above): out[i] is
 *     jpegqs_cuda_thumbnail_geometry's out_w x out_h.  Every box has left..bottom 0, scale_denom must
 *     be 1 (the scale is thumbnail's own), and filter is one of the five convolution filters.
 *   - Per sub-batch: every distinct draft scale is rendered by its own render call (at most four, more
 *     when smoothed and unsmoothed files, or CHW outputs that need neither stage, interleave); one reduce
 *     launch over the files with a factor above 1; the two resize launches over the files whose size
 *     changes.  A file that needs neither is stored by the render in the caller's layout.  The budget
 *     also counts each reduced picture.
 *   - Return.  As the mode call's; also JPEGQS_ERR_ARG with nothing done for a bad reducing_gap or
 *     thumbnail, a thumbnail box with an offset, or scale_denom other than 1 with thumbnail 1. */
int jpegqs_cuda_pixels_batch_reduced(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const int32_t *orientation, int mode, int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results, int thumbnail, double reducing_gap);

/* jpegqs_cuda_pixels_batch_jpeg_mode with thumbnail and reducing_gap as for pixels_batch_reduced: the
 * thumbnail (or reduced resize) is saved, progressive output included.  thumbnail 0 with reducing_gap
 * 0.0: byte for byte the mode call. */
int jpegqs_cuda_pixels_batch_jpeg_reduced(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len, const int32_t *orientation, int mode, int thumbnail, double reducing_gap);

/* The reduce of pixels_batch_reduced on the calling thread (host-only): Pillow's Image.reduce((factor_x,
 * factor_y), box) of a width x height x channels HWC picture (channels 1 or 3).  box: (left, top, right,
 * bottom) integers, or NULL for the whole picture.  out: ceil(box_w / factor_x) x ceil(box_h / factor_y)
 * x channels bytes, HWC.  Returns 0 or JPEGQS_ERR_ARG (NULL pointer, a factor below 1 or a cell of 2^23
 * samples or more, a box outside the picture or empty). */
int jpegqs_cuda_reduce_model(const uint8_t *src, int width, int height, int channels, int factor_x, int factor_y,
		const int32_t *box, uint8_t *out);

/* Steps 4 and 5 above on the calling thread (host-only), with the planning the batch uses: Pillow's
 * Image.resize((out_w, out_h), filter, box, reducing_gap) of a width x height x channels HWC picture.
 * box: (left, top, right, bottom) as doubles, as Pillow's Python layer holds it, or NULL for the whole
 * picture; reducing_gap 0.0 means None.  out: out_w x out_h x channels in layout HWC or CHW.  Returns 0
 * or JPEGQS_ERR_ARG (the checks of jpegqs_cuda_resize_model, a box outside the picture or empty, and the
 * refusals above). */
int jpegqs_cuda_resize_model_box(const uint8_t *src, int width, int height, int channels, int layout, int filter,
		const double *box, int out_w, int out_h, double reducing_gap, uint8_t *out);

/* ---- blur and sharpen: Pillow's ImageFilter.BoxBlur, GaussianBlur and UnsharpMask ----------------
 * Each channel byte is filtered on its own, in 32-bit unsigned integer arithmetic (libImaging BoxBlur.c
 * and UnsharpMask.c):
 *   - one box pass of radius R >= 0 along a line of n samples p, with r = (int)R,
 *     ww = (uint32)(2^24 / (float)(2R + 1)) in float, fw = (2^24 - (2r + 1) ww) / 2 and c(i) the index
 *     clamped to 0..n-1, gives (sum_{k=-r..r} p[c(x+k)] ww + (p[c(x-r-1)] + p[c(x+r+1)]) fw + 2^23) >> 24;
 *     every pass stores 8-bit samples;
 *   - BOX_BLUR (radius_x, radius_y): one pass along every row with radius_x, then one along every column
 *     with radius_y; an axis of radius 0 is skipped.  A negative radius is refused.
 *   - GAUSSIAN_BLUR (radius_x, radius_y): three row passes, then three column passes, with the box radius
 *     g(s) Pillow derives from the standard deviation s in float (sigma2 = s s / 3,
 *     L = sqrt(12 sigma2 + 1), l = floor((L - 1) / 2), g = l + (2l + 1)(l (l + 1) - 3 sigma2) /
 *     (6 (sigma2 - (l + 1)^2))); g(0) = 0 skips the axis, and a negative s acts as |s|.
 *   - UNSHARP_MASK (radius_x = radius_y = radius, percent, threshold): b = GAUSSIAN_BLUR(radius) of the
 *     input; per byte d = in - b, and the output is clamp(in + d * percent / 100, 0, 255) (C's truncating
 *     division) where |d| > threshold, else in.
 * Refused, because Pillow's 32-bit arithmetic would overflow: a radius (either axis, any kind) that is
 * not finite or whose magnitude is above JPEGQS_FILTER_MAX_RADIUS, and |percent| above
 * JPEGQS_FILTER_MAX_PERCENT (|d * percent| reaches 2^31).  percent and threshold are ignored by the
 * blurs. */
#define JPEGQS_FILTER_BOX_BLUR       1
#define JPEGQS_FILTER_GAUSSIAN_BLUR  2
#define JPEGQS_FILTER_UNSHARP_MASK   3
#define JPEGQS_FILTER_MAX_RADIUS     65535.0f
#define JPEGQS_FILTER_MAX_PERCENT    8421504
typedef struct jpegqs_cuda_image_filter {
	int32_t kind;                      /* JPEGQS_FILTER_* */
	float radius_x, radius_y;
	int32_t percent, threshold;        /* UNSHARP_MASK */
} jpegqs_cuda_image_filter;

/* jpegqs_cuda_pixels_batch_reduced, then filters[0..nfilters) applied in order to every file's picture:
 * file i is Pillow's [crop().resize() | thumbnail()].filter(F1).filter(F2)... of the picture the reduced
 * call gives.  The filter is the last stage: the earlier ones write HWC into the context's buffers and the
 * last filter pass writes out[i] in the caller's layout.  Per sub-batch and filter: one row launch over
 * the files whose rows (width x channels bytes) are at most 16384 bytes (every row pass fused in
 * shared memory), one launch per row pass over the wider ones, one launch per column pass over all.  The
 * budget counts three pictures of scratch per file.  nfilters 0 is byte for byte the reduced call.
 *   - Return.  As the reduced call's; also JPEGQS_ERR_ARG with nothing done for filters NULL with
 *     nfilters > 0, nfilters outside 0..64, or a filter refused above. */
int jpegqs_cuda_pixels_batch_filtered(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const int32_t *orientation, int mode, int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results, int thumbnail, double reducing_gap, const jpegqs_cuda_image_filter *filters,
		int nfilters);

/* jpegqs_cuda_pixels_batch_jpeg_reduced with filters as for pixels_batch_filtered: the filtered picture is
 * saved.  nfilters 0 is byte for byte the reduced call. */
int jpegqs_cuda_pixels_batch_jpeg_filtered(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len, const int32_t *orientation, int mode, int thumbnail, double reducing_gap,
		const jpegqs_cuda_image_filter *filters, int nfilters);

/* The filters of pixels_batch_filtered on the calling thread (host-only), through the same per-sample
 * functions and pass plan: filters[0..nfilters) applied in order to a width x height x channels HWC
 * picture (channels 1 or 3) into out (the same size, HWC; it may not overlap src).  Returns 0 or
 * JPEGQS_ERR_ARG (NULL pointer, bad size or channels, the refusals above). */
int jpegqs_cuda_image_filter_model(const uint8_t *src, int width, int height, int channels,
		const jpegqs_cuda_image_filter *filters, int nfilters, uint8_t *out);

/* ---- one image sharded by MCU rows over several GPUs (SURVEY.md 8e) ----------------------
 * Every rank - a device of this process, or another process on the same box - smooths one slab
 * of contiguous MCU rows and exchanges ONE pixel row per plane with each neighbour after every
 * IDCT pass (quantsmooth.h:1396-1401: a pass reads only start-of-pass neighbour pixels).  The
 * exchange runs inside CUDA kernels over peer memory (NVLink P2P / CUDA IPC mailboxes, sequence
 * numbers instead of events): no host round trip, no NCCL call on the data path.  The
 * reference's `stop` logic is evaluated on the device from flags the ranks OR-combine, so all
 * ranks issue the same schedule whatever their data.  Results are bit-identical to the
 * unsharded run for any rank count.
 *
 *   link_create on every rank -> link_export + (all-gather of the handles by the caller) +
 *   link_connect_ipc, or link_connect_local for the devices of one process -> run_slab, as often
 *   as wanted, by all ranks alike -> link_destroy.                                            */
typedef struct jpegqs_cuda_link jpegqs_cuda_link;
typedef struct {
	int32_t rank, world;
	uint32_t row0[JPEGQS_CUDA_MAX_COMP];        /* first block row of the slab inside component c  */
	uint32_t hblk_total[JPEGQS_CUDA_MAX_COMP];  /* block rows of the whole component               */
} jpegqs_cuda_slab;
/* max_wblk: widest component (in blocks) any later run will exchange */
int jpegqs_cuda_link_create(jpegqs_cuda_ctx *ctx, int rank, int world, uint32_t max_wblk, jpegqs_cuda_link **out);
void jpegqs_cuda_link_destroy(jpegqs_cuda_link *link);
int jpegqs_cuda_link_handle_bytes(void);
int jpegqs_cuda_link_export(jpegqs_cuda_link *link, void *handle);
int jpegqs_cuda_link_connect_ipc(jpegqs_cuda_link *link, const void *handles_in_rank_order);
int jpegqs_cuda_link_connect_local(jpegqs_cuda_link **links_in_rank_order, int world);
/* slab: the image with comp[].hblk = block rows held by this rank and coef / rows / coef_up
 * covering exactly those rows (host memory, or device memory with on_device != 0);
 * image_width / image_height are the WHOLE image's.  No progress callback.  link may be NULL
 * for world == 1.  Returns the reference's stop value (identical on every rank) or an error. */
int jpegqs_cuda_run_slab(jpegqs_cuda_ctx *ctx, jpegqs_cuda_link *link, jpegqs_cuda_image *slab,
		const jpegqs_cuda_slab *geom, int flags, int niter, int on_device, void *stream);

/* The devices of ONE process behind one call (what do_quantsmooth uses when JPEGQS_GPUS is
 * set): contexts + links for ndev devices (devices == NULL: ordinals 0..ndev-1; ndev <= 0: all),
 * one host thread per device inside run_host_multi.  An image is spread over as many devices as
 * it has waves of the smoothing kernel (JPEGQS_MIN_BLOCKS_PER_GPU luma blocks per device,
 * default 132*16*32, one wave on an H100), so a small image stays on device 0 with the slab-pipelined run_host. */
typedef struct jpegqs_cuda_multi jpegqs_cuda_multi;
int jpegqs_cuda_multi_create(int ndev, const int *devices, jpegqs_cuda_multi **out);
void jpegqs_cuda_multi_destroy(jpegqs_cuda_multi *m);
int jpegqs_cuda_multi_devices(const jpegqs_cuda_multi *m);
jpegqs_cuda_ctx *jpegqs_cuda_multi_ctx(jpegqs_cuda_multi *m, int i);
const char *jpegqs_cuda_multi_last_error(const jpegqs_cuda_multi *m);
int jpegqs_cuda_multi_plan(const jpegqs_cuda_multi *m, const jpegqs_cuda_image *img);   /* devices it would use */
/* host buffers / block-row tables like jpegqs_cuda_run_host; no progress callback */
int jpegqs_cuda_run_host_multi(jpegqs_cuda_multi *m, jpegqs_cuda_image *img, int flags, int niter);

/* ---- pass-level entry points (multi-GPU slabs: the caller exchanges halo rows between
 *      the passes; see DESIGN.md section 5).  All pointers are DEVICE pointers. ---------- */
typedef struct {
	int16_t *coef;             /* [hblk][wblk][64] of this slab                            */
	uint8_t *plane;            /* jpegqs_cuda_plane_bytes(wblk, hblk) bytes                */
	const uint8_t *plane2;     /* down-sampled luma plane of the same geometry, or NULL    */
	uint32_t wblk, hblk;       /* hblk = block rows held by this slab                      */
	uint16_t quant[64];        /* raw quantval                                             */
	int32_t luma;              /* !ci || colour space != YCbCr (quantsmooth.h:2639)        */
	int32_t top_edge;          /* slab touches the image top / bottom: replicate the       */
	int32_t bottom_edge;       /* border row there (2618-2619) instead of expecting a halo */
} jpegqs_cuda_job;

size_t jpegqs_cuda_plane_bytes(uint32_t wblk, uint32_t hblk);
int jpegqs_cuda_plane_stride(uint32_t wblk);
int jpegqs_cuda_plane_pad(void);   /* byte offset of pixel column 0 inside a plane row */

#define JPEGQS_PASS_DEQUANT 1      /* iteration 0: coef *= quantval, range check (2596-2603) */
#define JPEGQS_PASS_CLAMP   2      /* write coefficients back clamped to +-1023 (2670-2689)  */
/* IDCT pass (2589-2620): renders each job's plane (+ replicated borders).  *bad receives a
 * bit mask (bit i = job i, jobs >= 31 share bit 31) of the jobs in which a de-quantized
 * coefficient left [-2048, 2047] (host sync).  bad may be NULL. */
int jpegqs_cuda_pass_idct(jpegqs_cuda_ctx *ctx, int njobs, const jpegqs_cuda_job *jobs, int mode,
		int *bad, void *stream);
/* smoothing pass (2627-2640): quantsmooth_block on every block of every job */
int jpegqs_cuda_pass_smooth(jpegqs_cuda_ctx *ctx, int njobs, const jpegqs_cuda_job *jobs, int flags,
		int clamp_out, void *stream);

/* luma -> chroma hand-over for slabs (JOINT_YUV / UPSAMPLE_UV): the down-sampled luma plane
 * of quantsmooth.h:2753-2815 for one slab.  Rows are addressed inside the WHOLE component:
 * y_row0 / c_row0 = first luma / chroma block row of the slab, *_hblk_total = block rows of the
 * whole component.  Writes the slab's rows of plane2 (chroma slab geometry, c_rows block rows)
 * incl. the left/right border and, at an image edge, the replicated border rows; interior
 * halo rows (row -1 / row c_rows*8 of the slab) must be exchanged by the caller. */
int jpegqs_cuda_pass_downsample(jpegqs_cuda_ctx *ctx, const uint8_t *yplane, uint32_t y_wblk,
		uint32_t y_row0, uint32_t y_hblk_total, uint8_t *plane2, uint32_t c_wblk, uint32_t c_rows, uint32_t c_row0,
		uint32_t c_hblk_total, int ws, int hs, int top_edge, int bottom_edge, void *stream);
/* upsample_row + FDCT (quantsmooth.h:2691-2752) for one chroma component of one slab: fills
 * coef_up [y_rows][y_wblk][64]; scratch = y_wblk*8 * y_rows*8 bytes of device memory.  The
 * chroma plane and plane2 need valid halo rows (3x3 windows). */
int jpegqs_cuda_pass_upsample(jpegqs_cuda_ctx *ctx, const uint8_t *cplane, const uint8_t *plane2,
		uint32_t c_wblk, const uint8_t *yplane, uint32_t y_wblk, uint32_t y_rows, uint32_t y_row0,
		int16_t *coef_up, uint8_t *scratch, int ws, int hs, uint32_t image_width, uint32_t image_height,
		void *stream);

/* ---- decode to interleaved 8-bit RGB (SURVEY.md 8f row f2) -----------------------------
 * What libjpeg produces after the reference's jpegqs_start_decompress (quantsmooth.h:2880-2904):
 * islow IDCT, libjpeg's "fancy" chroma up-sampling (h2v1 / h2v2; other ratios: replication),
 * YCbCr -> RGB with libjpeg's fixed-point constants.  1 or 3 components.  Components whose
 * quant table is not all ones are de-quantized first, so the call also decodes an untouched
 * coefficient set.  rgb: image_width * image_height * 3 bytes (host, or device if on_device;
 * device coefficient arrays that still carry quant tables are de-quantized in place).  Unlike
 * jpegqs_cuda_render_async it does not check that the blocks cover the image. */
int jpegqs_cuda_render_rgb(jpegqs_cuda_ctx *ctx, const jpegqs_cuda_image *img, int on_device,
		uint8_t *rgb, void *stream);

/* ---- introspection used by the parity tests ------------------------------------------- */
/* the 64 weight tables exactly as the device consumes them but WITHOUT the power-of-two
 * pre-scale, natural coefficient order, 160 (or 272 with JPEGQS_DIAGONALS) floats each;
 * replaces quantsmooth_init (quantsmooth.h:251-301).  Returns floats per coefficient. */
int jpegqs_cuda_tables(int flags, float *out);
/* host evaluation of the device's exact-division helper (GET_ORIG_COEF, 324-341) */
int jpegqs_cuda_orig_coef(int coef, int q);
/* the smoothing kernel's chunk schedule for one quant table (host-only; DESIGN.md 3.3): the 63
 * AC coefficients in the reference's anti-diagonal visiting order (quantsmooth.h:313-322,
 * 1403-1409), grouped into chunks.  out: 12 bytes per chunk = {type, n, first, 0, idx[8]} with
 * type 0 = plain, 1 = the diagonal's two edge coefficients, 2 = equal quant values (shared
 * threshold work), 3 = mixed (n full coefficients, then the row-0 and the column-0 one: n + 2
 * indices); idx = natural-order coefficient indices.  uniform: bit 0 = uniform chunks, bit 1 =
 * mixed chunks; quant == NULL gives the table-independent schedule.  Returns the chunk count (<= 64), or JPEGQS_ERR_ARG. */
int jpegqs_cuda_chunk_schedule(const uint16_t *quant, int max_coefs, int uniform, uint8_t *out);
/* jpegqs_cuda_decode_async's algorithm run on the CPU, for one file: the same unstuffing, the same
 * subsequences of sub_bytes (tuning key 9) bytes, the same speculative decode, synchronisation rounds
 * (block rounds of 128 subsequences, one grid round, the in-order chain check), placement and final
 * decode, with the same block and unit decoders; threads run in sequence.  img->comp[c].coef are
 * HOST arrays.  *status receives the JPEGQS_DECODE_* bits.  overrun (may be NULL, overrun_cap
 * entries): per subsequence, in order, the units the synchronisation steps decoded past its end
 * before the chain from its exit met the speculative decode of the next subsequence (0 where it
 * met at once).  *nsub (may be NULL) receives the subsequence count.  Returns 0 or JPEGQS_ERR_ARG. */
int jpegqs_cuda_decode_model(const jpegqs_cuda_image *img, const jpegqs_cuda_scan *scan, const uint8_t *data,
		size_t data_len, int sub_bytes, int32_t *status, uint32_t *overrun, size_t overrun_cap, size_t *nsub);

#ifdef __cplusplus
}
#endif
#endif
