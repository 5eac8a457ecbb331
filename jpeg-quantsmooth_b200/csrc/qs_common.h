/*
 * qs_common.h - types shared by the host driver (qs_cuda.cu) and the sm_90a kernels
 * (qs_kernels.cu).  Nothing here is visible through the C ABI (include/jpegqs_cuda.h).
 */
#ifndef QS_COMMON_H
#define QS_COMMON_H

#include <stdint.h>

/* flag bits, numerically equal to the public JPEGQS_* enum (include/libjpegqs.h) */
#define QS_DIAGONALS 1
#define QS_JOINT_YUV 2
#define QS_UPSAMPLE_UV 4
#define QS_LOW_QUALITY 8
#define QS_NO_REBALANCE 16
#define QS_NO_REBALANCE_UV 32

/* Sample planes.  Pixel (x, y) of a component (or of a slab of it) lives at
 * plane[(y + 1) * stride + QS_PLANE_PAD + x]; row 0 / row h+1 and columns -1 / w are the
 * replicated 1-px border of reference quantsmooth.h:2612-2620 (or, at an interior slab
 * edge of a multi-GPU run, the neighbour's halo row).  stride = wblk*8 + 2*QS_PLANE_PAD. */
#define QS_PLANE_PAD 16
#define QS_PLANE_STRIDE(wblk) ((int)(wblk) * 8 + 2 * QS_PLANE_PAD)
#define QS_PLANE_BYTES(wblk, hblk) ((size_t)QS_PLANE_STRIDE(wblk) * ((size_t)(hblk) * 8 + 2))

/* Pixel differences enter the float pipeline pre-scaled by 2^-QS_SCALE_BITS (exact), the
 * weight tables pre-scaled by 2^(2*QS_SCALE_BITS); see DESIGN.md "exact rescaling". */
#define QS_SCALE_BITS 15

#define QS_TAB_PLAIN 160
#define QS_TAB_DIAG 272

/* chunk schedule of the 63 AC coefficients: 14 anti-diagonal groups (reverse zig-zag,
 * quantsmooth.h:313-322, 1403-1409) split into chunks of <= 4 coefficients that share the
 * pixel-difference work.  type 1 = the group's two edge coefficients (row 0: no vertical
 * terms; column 0: no horizontal terms; quantsmooth.h:1527, 1531); type 2 = a chunk whose
 * coefficients all have the same quant value, so t = max(R-|d|,0)^2 and a0 = d*t are
 * computed once per term and shared (3 + 5n FP ops per term instead of 8n); type 3 = "mixed":
 * n (1 or 2) full coefficients idx[0..n-1] plus the group's two edge coefficients idx[n] (row 0)
 * and idx[n+1] (column 0) in one chunk.  The schedule is built per quant table on the host
 * (qs_cuda.cu::build_chunks). */
typedef struct {
	uint8_t type, n, first, pad;
	uint8_t idx[8];
} QsChunk;
#define QS_MAX_CHUNKS 64

/* per-quant-table constants, device resident */
typedef struct {
	float Rs[64];        /* 2*q[i] * 2^-QS_SCALE_BITS  (range of quantsmooth.h:1406, scaled) */
	uint32_t m31[64];    /* ceil(2^31 / q[i]): exact floor-division magic, see qs_orig_coef */
	uint16_t q[64];      /* quantval with 0 -> 1 (quantsmooth.h:2508-2511) */
	uint16_t qraw[64];   /* raw quantval, used only by the iteration-0 dequantize (2598) */
	int32_t nchunks;     /* chunk schedule of this table */
	int32_t sched_slot;  /* index of the first table of this upload with the same schedule */
	QsChunk chunks[QS_MAX_CHUNKS];
} QsQuantDev;

/* one component (or one slab of block rows of it) taking part in a launch */
typedef struct {
	int16_t *coef;           /* [hblk][wblk][64] */
	uint8_t *plane;          /* sample plane of this component */
	const uint8_t *plane2;   /* down-sampled luma plane (JOINT_YUV predictor) or NULL */
	const QsQuantDev *quant;
	int32_t wblk, hblk;      /* blocks; hblk = rows present in this slab */
	int32_t stride;          /* bytes per plane row */
	int32_t nblocks;         /* wblk * hblk */
	int32_t tile_begin;      /* first 32-block tile of this job inside the launch */
	int32_t luma;            /* rebalance class (quantsmooth.h:2639) */
	int32_t top_edge;        /* 1: slab top is the image top -> replicate row -1 */
	int32_t bottom_edge;     /* 1: slab bottom is the image bottom */
	int32_t bad_slot;        /* index into the "coefficient out of range" flags */
	/* Device-side stop handling (sharded runs, qs_cuda.cu run_slab): bad_slot is then the
	 * component's slot in flags that live for the whole run, bad_first the slot of component 0 of
	 * the same image, and the kernels decide by themselves what the reference's `stop` logic
	 * (quantsmooth.h:2504, 2551-2566, 2602-2610) leaves to do: 0 = smooth, 1 = this component
	 * overflowed (clamp only), 2 = an earlier one did (de-quantize only).  stop_aware = 0: the
	 * host has already sorted that out (run_images, and every job built by qs_cuda.cu make_job
	 * unless run_job is given the run's flags). */
	int32_t bad_first, stop_aware;
} QsJob;

/* sharded runs: ranks exchange pixel rows and the out-of-range masks through mailboxes in peer
 * memory (NVLink P2P, or CUDA IPC between processes); see qs_kernels.cu qs_xchg_*_kernel */
#define QS_MAX_RANKS 16
#define QS_XCHG_SLOTS 12          /* planes per exchange: MAX_COMPONENTS + the down-sampled luma */
#define QS_XCHG_MAX_ROWS (2 * QS_XCHG_SLOTS)
typedef struct { const uint8_t *src; uint8_t *dst; uint32_t bytes, pad; } QsXchgRow;
typedef struct {
	QsXchgRow rows[QS_XCHG_MAX_ROWS]; int32_t nrows;
	uint32_t seq;
	uint32_t *flag[2];                       /* the neighbours' "rows have arrived" words (or NULL) */
	const int32_t *bad_src; int32_t bad_n;   /* out-of-range flags of this rank -> every peer */
	int32_t npeers;
	uint32_t *bad_dst[QS_MAX_RANKS], *bad_flag[QS_MAX_RANKS];
} QsXchgPush;
typedef struct {
	QsXchgRow rows[QS_XCHG_MAX_ROWS]; int32_t nrows;
	uint32_t seq;
	const uint32_t *flag[2];                 /* this rank's "rows have arrived" words to wait for */
	int32_t *bad_io; int32_t bad_n;          /* local flags, OR-ed with every peer's message */
	int32_t npeers;
	const uint32_t *bad_in[QS_MAX_RANKS], *bad_flag[QS_MAX_RANKS];
	int32_t *timeout_flag;                   /* mapped host word set if a peer never signalled */
} QsXchgPull;

#define QS_MAX_JOBS 1024

/* IDCT-pass modes */
#define QS_IDCT_DEQUANT 1     /* multiply by qraw, range-check (iteration 0) */
#define QS_IDCT_CLAMP 2       /* write coefficients back clamped to +-1023 (2670-2689) */
#define QS_IDCT_NOPLANE 4     /* do not render pixels (dequantize/clamp only) */

#endif
