/*
 * qs_kernels.cu - hand-written sm_90a (Hopper) kernels for the jpeg-quantsmooth coefficient
 * smoothing path.  Compile with -gencode arch=compute_90a,code=sm_90a -fmad=false.
 *
 * Mapping (DESIGN.md section 3): ONE THREAD PER 8x8 BLOCK.  The reference's per-coefficient
 * sums a2/a3 (reference quantsmooth.h:1517-1545) must be accumulated sequentially in the
 * scalar loop order with separately rounded mul/add to be bit-exact, so a block is never
 * split across lanes; a warp runs 32 blocks through the same (coefficient, term) sequence,
 * which makes every weight-table read warp-uniform (shared-memory broadcast) and keeps all
 * 32 FP32 lanes busy.  The path is FP32-issue bound (SURVEY.md 8d), not HBM bound.
 *
 * Kernels:
 *   qs_idct_pass_kernel   dequantize (iteration 0) + islow IDCT -> sample plane + borders
 *                         (reference quantsmooth.h:2589-2620, idct.h:57-548)
 *   qs_smooth_kernel      quantsmooth_block for every block of every job
 *                         (reference quantsmooth.h:564-1849 scalar branches)
 *   qs_downsample_kernel  box-downsampled luma plane (quantsmooth.h:2753-2815)
 *   qs_upsample_kernel    upsample_row (quantsmooth.h:1851-2394 scalar branches)
 *   qs_fdct_plane_kernel  float FDCT of the up-sampled chroma plane (quantsmooth.h:2735-2750)
 *   qs_scale_clamp_kernel dequantize-only / clamp-only fallbacks (quantsmooth.h:2551-2566, 2670-2689)
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <limits.h>
#include <string.h>
#include <type_traits>
#include <vector>
#include "qs_common.h"
#include "qs_kernels.h"

/* Phase clocks (measurement builds only, -DQS_PHASE_CLOCKS): every warp accumulates the SM
 * clock cycles it spends in each phase of the smoothing kernel into shared memory and adds them
 * to qs_phase_acc at the end; read back with qs_read_phase_clocks.  In lock step the four warps
 * of a sub-partition are in the same phase, so cycles/4 per phase is sub-partition time. */
#ifdef QS_PHASE_CLOCKS
#define QS_NPHASE 16
__device__ unsigned long long qs_phase_acc[QS_NPHASE];
struct QsPh {
	uint32_t t; uint32_t *acc;
	__device__ __forceinline__ void start(uint32_t *a) { acc = a; t = (uint32_t)clock(); }
	__device__ __forceinline__ void mark(int k) { uint32_t n = (uint32_t)clock(); acc[k] += n - t; t = n; }
};
#define QS_PH_MARK(ph, k) (ph).mark(k)
#else
struct QsPh {};
#define QS_PH_MARK(ph, k) ((void)0)
#endif

/* table-independent schedule: used by a lock-step group whose warps work on components with
 * different schedules (their barrier sequences must match) */
__device__ QsChunk d_chunks[QS_MAX_CHUNKS];
__device__ int d_nchunks;

/* ------------------------------------------------------------------------------------------
 * small helpers
 * ------------------------------------------------------------------------------------------ */
__device__ __forceinline__ int qs_find_job(const QsJob *__restrict__ jobs, int njobs, int tile) {
	int lo = 0, hi = njobs - 1;
	while (lo < hi) {                       /* last job with tile_begin <= tile */
		int mid = (lo + hi + 1) >> 1;
		if (__ldg(&jobs[mid].tile_begin) <= tile) lo = mid; else hi = mid - 1;
	}
	return lo;
}

/* what the reference's `stop` logic leaves to do for this job (see QsJob.stop_aware) */
__device__ __forceinline__ int qs_job_state(const QsJob *job, const int *__restrict__ bad) {
	if (!bad || !job->stop_aware) return 0;
	for (int s = job->bad_first; s < job->bad_slot; s++) if (*(const volatile int *)&bad[s]) return 2;
	return *(const volatile int *)&bad[job->bad_slot] ? 1 : 0;
}

/* a0 = round_half_away(c / q) * q  (reference quantsmooth.h:338-341 plain form; the
 * reference's reciprocal form 324-337 is equal on the valid range, SURVEY.md 8a8).
 * m31 = ceil(2^31 / q) makes floor((|c| + q/2) / q) one IMAD.HI; exact while
 * |c| + q/2 < 2^31 / q, i.e. for all q < 2^11 and |c| < 2^16. */
__host__ __device__ __forceinline__ int qs_orig_coef(int c, int q, uint32_t m31) {
	uint32_t mag = (uint32_t)(c < 0 ? -c : c) + (uint32_t)(q >> 1);
#ifdef __CUDA_ARCH__
	int k = (int)__umulhi(mag << 1, m31);
#else
	int k = (int)(((uint64_t)(mag << 1) * m31) >> 32);
#endif
	int a0 = k * q;
	return c < 0 ? -a0 : a0;
}

extern "C" int qs_host_orig_coef(int c, int q) {
	uint32_t m31 = (uint32_t)(((1ull << 31) + (uint32_t)q - 1) / (uint32_t)q);
	return qs_orig_coef(c, q, m31);
}

/* x86 cvttss2si semantics: NaN / out of range -> INT_MIN (SURVEY.md 7.3 item 2) */
__device__ __forceinline__ int qs_cvtt_x86(float x) {
	return fabsf(x) < 2147483648.0f ? __float2int_rz(x) : INT_MIN;
}

/* ------------------------------------------------------------------------------------------
 * integer islow IDCT (reference idct.h:39-89 butterfly, 469-538 passes)
 * ------------------------------------------------------------------------------------------ */
/* RND: rounding constant of the descale that follows (idct.h:469-538: +1024 before >> 11 in
 * pass 1, +(257 << 17) before >> 18 in pass 2).  Every output is e_j +- t_k with e_j containing
 * exactly one of t0/t1 below, so adding RND there once is the same integer sum as adding it to
 * each of the eight outputs - and it is free inside the IMAD that forms (in0 +- in4) << 13. */
template <int RND>
__host__ __device__ __forceinline__ void qs_islow_1d(const int *in, int *out) {
	int z1, z2, z3, z4, z5, e0, e1, e2, e3, t0, t1, t2, t3, a, b;
	z2 = in[2]; z3 = in[6];
	z1 = (z2 + z3) * 4433;
	a = z1 - z3 * 15137; b = z1 + z2 * 6270;
	t0 = (in[0] + in[4]) * 8192 + RND; t1 = (in[0] - in[4]) * 8192 + RND;
	e0 = t0 + b; e3 = t0 - b; e1 = t1 + a; e2 = t1 - a;
	t0 = in[7]; t1 = in[5]; t2 = in[3]; t3 = in[1];
	z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2; z4 = t1 + t3;
	z5 = (z3 + z4) * 9633;
	t0 *= 2446; t1 *= 16819; t2 *= 25172; t3 *= 12299;
	z1 *= 7373; z2 *= 20995; z3 *= 16069; z4 *= 3196;
	z3 = z5 - z3; z4 = z5 - z4;
	t0 += z3 - z1; t1 += z4 - z2; t2 += z3 - z2; t3 += z4 - z1;
	/* (forming the outputs as three-input sums e0 +- b +- t3 - fewer instructions, IADD3 on the
	 * ALU pipe - was measured slower in the refresh IDCTs) */
	out[0] = e0 + t3; out[7] = e0 - t3; out[1] = e1 + t2; out[6] = e1 - t2;
	out[2] = e2 + t1; out[5] = e2 - t1; out[3] = e3 + t0; out[4] = e3 - t0;
}

/* four int32 -> four saturated bytes b0 | b1<<8 | b2<<16 | b3<<24 */
__host__ __device__ __forceinline__ uint32_t qs_pack_sat_u8(int b0, int b1, int b2, int b3) {
#ifdef __CUDA_ARCH__
	uint32_t t, r;
	asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, 0;" : "=r"(t) : "r"(b3), "r"(b2));
	asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(b1), "r"(b0), "r"(t));
	return r;
#else
	const int b[4] = {b0, b1, b2, b3};
	uint32_t r = 0;
	for (int k = 0; k < 4; k++) r |= (uint32_t)(b[k] < 0 ? 0 : b[k] > 255 ? 255 : b[k]) << (8 * k);
	return r;
#endif
}

/* second pass over a 64-int workspace (already column-transformed and descaled):
 * rows -> packed pixels lo[y] = px[y][0..3], hi[y] = px[y][4..7] */
__host__ __device__ __forceinline__ void qs_islow_rows(const int *ws, uint32_t *lo, uint32_t *hi) {
#pragma unroll
	for (int y = 0; y < 8; y++) {
		int o[8];
		qs_islow_1d<(257 << 17)>(ws + y * 8, o);
#pragma unroll
		for (int k = 0; k < 8; k++) o[k] >>= 18;
		/* clamp to [0,255] and pack: one saturating I2IP per two pixels (idct.h:509-511) */
		lo[y] = qs_pack_sat_u8(o[0], o[1], o[2], o[3]);
		hi[y] = qs_pack_sat_u8(o[4], o[5], o[6], o[7]);
	}
}

/* column x of the block: bytes px[0..3][x], px[4..7][x] */
__device__ __forceinline__ uint2 qs_gather_col(const uint32_t *w, int byte) {
	uint32_t s = 0x4440u | (uint32_t)byte | ((uint32_t)(4 + byte) << 4);   /* [w0.b, w1.b, -, -] */
	uint32_t t01 = __byte_perm(w[0], w[1], s), t23 = __byte_perm(w[2], w[3], s);
	uint32_t t45 = __byte_perm(w[4], w[5], s), t67 = __byte_perm(w[6], w[7], s);
	return make_uint2(__byte_perm(t01, t23, 0x5410), __byte_perm(t45, t67, 0x5410));
}

/* ------------------------------------------------------------------------------------------
 * float FDCT, order-exact (reference idct.h:608-628 op list, 896-915 passes)
 * ------------------------------------------------------------------------------------------ */
#define FA(a, b) __fadd_rn(a, b)
#define FS(a, b) __fsub_rn(a, b)
#define FM(a, b) __fmul_rn(a, b)

__device__ __forceinline__ void qs_fdct_1d(const float *in, float *r) {
	float t0, t1, t2, t3, t4, t5, t6, t7, z1, z2, z3, z4, z5;
	t0 = FA(in[0], in[7]); t7 = FS(in[0], in[7]);
	t1 = FA(in[1], in[6]); t6 = FS(in[1], in[6]);
	t2 = FA(in[2], in[5]); t5 = FS(in[2], in[5]);
	t3 = FA(in[3], in[4]); t4 = FS(in[3], in[4]);
	z1 = FA(t0, t3); z4 = FS(t0, t3); z2 = FA(t1, t2); z3 = FS(t1, t2);
	r[0] = FA(z1, z2); r[4] = FS(z1, z2);
	z1 = FM(FA(z3, z4), 0.541196100f);
	r[2] = FA(z1, FM(z4, 0.765366865f));
	r[6] = FS(z1, FM(z3, 1.847759065f));
	z1 = FA(t4, t7); z2 = FA(t5, t6); z3 = FA(t4, t6); z4 = FA(t5, t7);
	z5 = FM(FA(z3, z4), 1.175875602f);
	t4 = FM(t4, 0.298631336f); t5 = FM(t5, 2.053119869f);
	t6 = FM(t6, 3.072711026f); t7 = FM(t7, 1.501321110f);
	z1 = FM(z1, 0.899976223f); z2 = FM(z2, 2.562915447f);
	z3 = FS(FM(z3, 1.961570560f), z5);
	z4 = FS(FM(z4, 0.390180644f), z5);
	r[7] = FS(t4, FA(z1, z3)); r[5] = FS(t5, FA(z2, z4));
	r[3] = FS(t6, FA(z2, z3)); r[1] = FS(t7, FA(z1, z4));
}

/* in-place 8x8: columns unscaled, then rows x0.125 */
__device__ __forceinline__ void qs_fdct_8x8(float *f) {
#pragma unroll
	for (int x = 0; x < 8; x++) {
		float in[8], r[8];
#pragma unroll
		for (int k = 0; k < 8; k++) in[k] = f[k * 8 + x];
		qs_fdct_1d(in, r);
#pragma unroll
		for (int k = 0; k < 8; k++) f[k * 8 + x] = r[k];
	}
#pragma unroll
	for (int y = 0; y < 8; y++) {
		float r[8];
		qs_fdct_1d(f + y * 8, r);
#pragma unroll
		for (int k = 0; k < 8; k++) f[y * 8 + k] = FM(r[k], 0.125f);
	}
}

/* 3x3 luma/chroma regression, weights 4/2/1 (reference quantsmooth.h:894-913, 2134-2155).
 * A = down-sampled luma, B = chroma, both pointing at the centre pixel. */
__device__ __forceinline__ float qs_regress(const uint8_t *__restrict__ A, const uint8_t *__restrict__ B,
		int stride, int &sA, int &sB) {
	int a, b, sAA, sAB;
#define TAP(dx, dy) a = A[(dy) * stride + (dx)]; b = B[(dy) * stride + (dx)]; \
	sA += a; sAA += a * a; sB += b; sAB += a * b;
	sA = sB = sAA = sAB = 0;
	TAP(0, 0) sA *= 2; sB *= 2; sAA *= 2; sAB *= 2;
	TAP(0, -1) TAP(-1, 0) TAP(1, 0) TAP(0, 1) sA *= 2; sB *= 2; sAA *= 2; sAB *= 2;
	TAP(-1, -1) TAP(1, -1) TAP(-1, 1) TAP(1, 1)
#undef TAP
	sAA = sAA * 16 - sA * sA;
	sAB = sAB * 16 - sA * sB;
	float scale = (float)sAA;
	if (sAA) scale = __fdiv_rn((float)sAB, scale);
	scale = scale < -16.0f ? -16.0f : scale;
	scale = scale > 16.0f ? 16.0f : scale;
	return scale;
}

#ifndef QS_IDCT_COALESCED
/* K1 as shipped: thread-private int4 loads at a 128-byte lane stride (the eight loads of a lane
 * walk one 128-byte line, which L1 keeps), register cap raised to allow 16 warps per SM.  The
 * shared-memory-transposed variant below (make variant DEFS=-DQS_IDCT_COALESCED) was measured
 * slower at 8, 16 and 24 warps per SM: the transposition costs more than the uncoalesced
 * requests.  Neither has been timed on an H100 yet. */
#ifndef QS_IDCT_MINB
#define QS_IDCT_MINB 2
#endif
#define QS_IDCT_THREADS 256
/* ------------------------------------------------------------------------------------------
 * K1: IDCT pass.  One thread per block; lanes of a warp own 32 consecutive blocks, so the
 * eight 8-byte row stores of a warp cover 256 contiguous bytes per pixel row.
 * ------------------------------------------------------------------------------------------ */
__global__ void __launch_bounds__(256, QS_IDCT_MINB) qs_idct_pass_kernel(const QsJob *__restrict__ jobs, int njobs,
		int total_tiles, int mode, int *__restrict__ bad_flags) {
	int tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
	if (tile >= total_tiles) return;
	int lane = threadIdx.x & 31;
	const QsJob *job = jobs + qs_find_job(jobs, njobs, tile);
	if (!(mode & QS_IDCT_DEQUANT) && qs_job_state(job, bad_flags)) return;
	int b = (tile - job->tile_begin) * 32 + lane;
	if (b >= job->nblocks) return;
	int W = job->wblk, H = job->hblk, stride = job->stride;
	int by = b / W, bx = b - by * W;
	int16_t *cptr = job->coef + (size_t)b * 64;
	const QsQuantDev *qd = job->quant;

	int c[64];
	{
		const int4 *p = (const int4 *)cptr;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			int4 v = p[j];
			c[j * 8 + 0] = (short)(v.x & 0xffff); c[j * 8 + 1] = v.x >> 16;
			c[j * 8 + 2] = (short)(v.y & 0xffff); c[j * 8 + 3] = v.y >> 16;
			c[j * 8 + 4] = (short)(v.z & 0xffff); c[j * 8 + 5] = v.z >> 16;
			c[j * 8 + 6] = (short)(v.w & 0xffff); c[j * 8 + 7] = v.w >> 16;
		}
	}
	if (mode & QS_IDCT_DEQUANT) {                       /* quantsmooth.h:2596-2603 */
		int val = 0;
#pragma unroll
		for (int k = 0; k < 64; k++) {
			int t = c[k] * (int)__ldg(&qd->qraw[k]);
			val |= t + 0x800;
			c[k] = (short)t;
		}
		if (val >> 12) atomicOr(&bad_flags[job->bad_slot], 1);
	}

	if (!(mode & QS_IDCT_NOPLANE)) {
		int ws[64];
#pragma unroll
		for (int x = 0; x < 8; x++) {
			int in[8], o[8];
#pragma unroll
			for (int k = 0; k < 8; k++) in[k] = c[k * 8 + x];
			qs_islow_1d<1024>(in, o);
#pragma unroll
			for (int k = 0; k < 8; k++) ws[k * 8 + x] = o[k] >> 11;
		}
		uint32_t lo[8], hi[8];
		qs_islow_rows(ws, lo, hi);

		uint8_t *p = job->plane + (size_t)(by * 8 + 1) * stride + QS_PLANE_PAD + bx * 8;
#pragma unroll
		for (int y = 0; y < 8; y++) *(uint2 *)(p + (size_t)y * stride) = make_uint2(lo[y], hi[y]);
		/* replicated borders, quantsmooth.h:2612-2620 */
		bool left = bx == 0, right = bx == W - 1;
		if (left) {
#pragma unroll
			for (int y = 0; y < 8; y++) p[(size_t)y * stride - 1] = (uint8_t)(lo[y] & 0xff);
		}
		if (right) {
#pragma unroll
			for (int y = 0; y < 8; y++) p[(size_t)y * stride + 8] = (uint8_t)(hi[y] >> 24);
		}
		if (by == 0 && job->top_edge) {
			uint8_t *r = p - stride;
			*(uint2 *)r = make_uint2(lo[0], hi[0]);
			if (left) r[-1] = (uint8_t)(lo[0] & 0xff);
			if (right) r[8] = (uint8_t)(hi[0] >> 24);
		}
		if (by == H - 1 && job->bottom_edge) {
			uint8_t *r = p + (size_t)8 * stride;
			*(uint2 *)r = make_uint2(lo[7], hi[7]);
			if (left) r[-1] = (uint8_t)(lo[7] & 0xff);
			if (right) r[8] = (uint8_t)(hi[7] >> 24);
		}
	}

	if (mode & (QS_IDCT_DEQUANT | QS_IDCT_CLAMP)) {
		if (mode & QS_IDCT_CLAMP) {                     /* quantsmooth.h:2670-2689 */
#pragma unroll
			for (int k = 0; k < 64; k++) c[k] = min(max(c[k], -1023), 1023);
		}
		int4 *p = (int4 *)cptr;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			int4 v;
			v.x = (c[j * 8 + 0] & 0xffff) | (c[j * 8 + 1] << 16);
			v.y = (c[j * 8 + 2] & 0xffff) | (c[j * 8 + 3] << 16);
			v.z = (c[j * 8 + 4] & 0xffff) | (c[j * 8 + 5] << 16);
			v.w = (c[j * 8 + 6] & 0xffff) | (c[j * 8 + 7] << 16);
			p[j] = v;
		}
	}
}

#else
/* ------------------------------------------------------------------------------------------
 * K1, coalesced variant: a warp owns 32 consecutive blocks = 4 KB of contiguous coefficients and
 * moves them with eight fully coalesced 512-byte requests (4 cache lines per request instead of
 * the 32 that per-thread loads at a 128-byte lane stride touch: no LSU queue pressure), staged in
 * shared memory as 16-byte chunks in 128-byte rows with the chunk index XOR-ed by the row
 * number - the 8 lanes of a quarter warp then hit 8 different chunk columns both when the tile is
 * stored (one row, chunks 0..7) and when every lane fetches its own block (8 rows, one chunk
 * each): conflict-free 128-bit shared accesses, 8 STS.128 + 8 LDS.128 per thread.
 * ------------------------------------------------------------------------------------------ */
#ifndef QS_IDCT_MINB
#define QS_IDCT_MINB 2
#endif
#define QS_IDCT_THREADS 256
__global__ void __launch_bounds__(QS_IDCT_THREADS, QS_IDCT_MINB) qs_idct_pass_kernel(const QsJob *__restrict__ jobs,
		int njobs, int total_tiles, int mode, int *__restrict__ bad_flags) {
	__shared__ int4 sm[QS_IDCT_THREADS / 32][32 * 8];
	int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	int tile = blockIdx.x * (QS_IDCT_THREADS / 32) + warp;
	if (tile >= total_tiles) return;                    /* whole warps leave: only __syncwarp below */
	const QsJob *job = jobs + qs_find_job(jobs, njobs, tile);
	if (!(mode & QS_IDCT_DEQUANT) && qs_job_state(job, bad_flags)) return;
	int b0 = (tile - job->tile_begin) * 32;
	int nb = min(32, job->nblocks - b0);
	int4 *sw = sm[warp];
	int4 *g = (int4 *)(job->coef + (size_t)b0 * 64);
#pragma unroll
	for (int j = 0; j < 8; j++) {
		int P = j * 32 + lane, blk = P >> 3;            /* 16-byte chunk P of the tile: block P/8, chunk P%8 */
		if (blk < nb) sw[blk * 8 + ((P & 7) ^ (blk & 7))] = g[P];
	}
	__syncwarp();
	const bool valid = lane < nb;
	int W = job->wblk, H = job->hblk, stride = job->stride;
	int b = b0 + (valid ? lane : 0);
	int by = b / W, bx = b - by * W;
	const QsQuantDev *qd = job->quant;

	if (valid) {
		int c[64];
#pragma unroll
		for (int j = 0; j < 8; j++) {
			int4 v = sw[lane * 8 + (j ^ (lane & 7))];
			c[j * 8 + 0] = (short)(v.x & 0xffff); c[j * 8 + 1] = v.x >> 16;
			c[j * 8 + 2] = (short)(v.y & 0xffff); c[j * 8 + 3] = v.y >> 16;
			c[j * 8 + 4] = (short)(v.z & 0xffff); c[j * 8 + 5] = v.z >> 16;
			c[j * 8 + 6] = (short)(v.w & 0xffff); c[j * 8 + 7] = v.w >> 16;
		}
		if (mode & QS_IDCT_DEQUANT) {                       /* quantsmooth.h:2596-2603 */
			int val = 0;
#pragma unroll
			for (int k = 0; k < 64; k++) {
				int t = c[k] * (int)__ldg(&qd->qraw[k]);
				val |= t + 0x800;
				c[k] = (short)t;
			}
			if (val >> 12) atomicOr(&bad_flags[job->bad_slot], 1);
		}
		if (!(mode & QS_IDCT_NOPLANE)) {
			int ws[64];
#pragma unroll
			for (int x = 0; x < 8; x++) {
				int in[8], o[8];
#pragma unroll
				for (int k = 0; k < 8; k++) in[k] = c[k * 8 + x];
				qs_islow_1d<1024>(in, o);
#pragma unroll
				for (int k = 0; k < 8; k++) ws[k * 8 + x] = o[k] >> 11;
			}
			uint32_t lo[8], hi[8];
			qs_islow_rows(ws, lo, hi);
			uint8_t *p = job->plane + (size_t)(by * 8 + 1) * stride + QS_PLANE_PAD + bx * 8;
#pragma unroll
			for (int y = 0; y < 8; y++) *(uint2 *)(p + (size_t)y * stride) = make_uint2(lo[y], hi[y]);
			/* replicated borders, quantsmooth.h:2612-2620 */
			bool left = bx == 0, right = bx == W - 1;
			if (left) {
#pragma unroll
				for (int y = 0; y < 8; y++) p[(size_t)y * stride - 1] = (uint8_t)(lo[y] & 0xff);
			}
			if (right) {
#pragma unroll
				for (int y = 0; y < 8; y++) p[(size_t)y * stride + 8] = (uint8_t)(hi[y] >> 24);
			}
			if (by == 0 && job->top_edge) {
				uint8_t *r = p - stride;
				*(uint2 *)r = make_uint2(lo[0], hi[0]);
				if (left) r[-1] = (uint8_t)(lo[0] & 0xff);
				if (right) r[8] = (uint8_t)(hi[0] >> 24);
			}
			if (by == H - 1 && job->bottom_edge) {
				uint8_t *r = p + (size_t)8 * stride;
				*(uint2 *)r = make_uint2(lo[7], hi[7]);
				if (left) r[-1] = (uint8_t)(lo[7] & 0xff);
				if (right) r[8] = (uint8_t)(hi[7] >> 24);
			}
		}
		if (mode & (QS_IDCT_DEQUANT | QS_IDCT_CLAMP)) {
			if (mode & QS_IDCT_CLAMP) {                     /* quantsmooth.h:2670-2689 */
#pragma unroll
				for (int k = 0; k < 64; k++) c[k] = min(max(c[k], -1023), 1023);
			}
#pragma unroll
			for (int j = 0; j < 8; j++) {
				int4 v;
				v.x = (c[j * 8 + 0] & 0xffff) | (c[j * 8 + 1] << 16);
				v.y = (c[j * 8 + 2] & 0xffff) | (c[j * 8 + 3] << 16);
				v.z = (c[j * 8 + 4] & 0xffff) | (c[j * 8 + 5] << 16);
				v.w = (c[j * 8 + 6] & 0xffff) | (c[j * 8 + 7] << 16);
				sw[lane * 8 + (j ^ (lane & 7))] = v;
			}
		}
	}
	if (mode & (QS_IDCT_DEQUANT | QS_IDCT_CLAMP)) {         /* coefficients back, coalesced */
		__syncwarp();
#pragma unroll
		for (int j = 0; j < 8; j++) {
			int P = j * 32 + lane, blk = P >> 3;
			if (blk < nb) g[P] = sw[blk * 8 + ((P & 7) ^ (blk & 7))];
		}
	}
}
#endif

/* ------------------------------------------------------------------------------------------
 * K2: the smoothing pass.
 *
 * Persistent CTAs (one per SM, 16 warps), dynamic tile scheduler (one atomic per 32-block
 * tile).  Shared memory: the weight tables (40 KB, or 68 KB with DIAGONALS; read with
 * warp-uniform LDS.128 = broadcast) + per warp a private 7.5 KB region holding, for each of
 * the 32 lanes' blocks, the 64 coefficients (packed int16 pairs) and 14 packed 8-pixel words:
 *   words 0-7  rows of the block's current pixels ("buf", quantsmooth.h:1408)
 *   word  8/9  column 0 / column 7 of the block
 *   word 10-13 the 8 neighbour pixels above / below / left / right ("border", 1396-1401)
 * All per-lane arrays are [item][lane] so lanes hit consecutive banks.
 *
 * Exact rescaling: a pixel byte p is turned into the float 1 + p*2^-15 by one PRMT, so a
 * difference of two of them is d*2^-15 exactly; with R' = 2q*2^-15 the clamp max(R-|d|,0)
 * becomes ONE add.sat (result < 1, so only the lower clamp acts).  Squares and products
 * carry pure power-of-two factors which commute with IEEE rounding (no overflow/underflow
 * in range, DESIGN.md 3.3); the weight table is pre-multiplied by 2^30 so a1 and a3 are
 * bit-identical to the reference's, a2 comes out scaled by 2^-45 and is rescaled (exactly)
 * after the division.  Per (term, coefficient): 1 FADD.SAT + 5 FMUL + 2 FADD, no FMA.
 * ------------------------------------------------------------------------------------------ */
#define QS_SMOOTH_THREADS 512               /* default: 4 warps per sub-partition */
#define QS_WARP_MSUM (32 * 32 + 14 * 32 * 2)      /* word offset of the rebalance sums: 2 x int64 per lane */
#define QS_WARP_WORDS (QS_WARP_MSUM + 4 * 32)     /* uint32 words per warp region */

__device__ __forceinline__ float qs_px(uint32_t w, int j) {
	return __uint_as_float(__byte_perm(w, 0x3F800000u, 0x7604u | (uint32_t)(j << 4)));
}
__device__ __forceinline__ void qs_unpack8(uint2 w, float *f) {
	f[0] = qs_px(w.x, 0); f[1] = qs_px(w.x, 1); f[2] = qs_px(w.x, 2); f[3] = qs_px(w.x, 3);
	f[4] = qs_px(w.y, 0); f[5] = qs_px(w.y, 1); f[6] = qs_px(w.y, 2); f[7] = qs_px(w.y, 3);
}

/* CORE of reference quantsmooth.h:1519-1520 on scaled operands; nad = -|ds| */
__device__ __forceinline__ void qs_term(float ds, float nad, float w, float Rs, float &a2, float &a3) {
	float t;
	asm("add.rn.sat.f32 %0, %1, %2;" : "=f"(t) : "f"(Rs), "f"(nad));
	t = FM(t, t);
	float a0 = FM(ds, t);
	float a1 = FM(w, t);
	a2 = FA(a2, FM(a0, a1));
	a3 = FA(a3, FM(a1, a1));
}

/* one pixel of a packed row: word 0 = pixels 0..3, word 1 = pixels 4..7 */
__device__ __forceinline__ float qs_px8(uint2 w, int j) { return j < 4 ? qs_px(w.x, j) : qs_px(w.y, j - 4); }

/* All terms of one row step for the N coefficients of a chunk.  `prep(c)` is called after each
 * coefficient's terms: it expands a slice of the NEXT row's pixels, so the PRMTs (ALU pipe,
 * half rate) are interleaved with the FP work instead of forming a burst at the loop end
 * where, in lock step, all four warps of the sub-partition would queue on the ALU pipe. */
template <int N, int NT, bool UNI, class Prep>
__device__ __forceinline__ void qs_terms_row(const float *d, const float *const *tab, int off,
		const float *Rs, float *a2, float *a3, Prep prep) {
	float nad[8], t[8], a0[8];
#pragma unroll
	for (int x = 0; x < NT; x++) nad[x] = -fabsf(d[x]);
	if (UNI) {
		/* all coefficients of the chunk share the quant value: t and a0 = d*t are the same
		 * numbers for each of them, computed once (identical roundings, so still bit-exact) */
#pragma unroll
		for (int x = 0; x < NT; x++) {
			asm("add.rn.sat.f32 %0, %1, %2;" : "=f"(t[x]) : "f"(Rs[0]), "f"(nad[x]));
			t[x] = FM(t[x], t[x]);
			a0[x] = FM(d[x], t[x]);
		}
	}
#pragma unroll
	for (int c = 0; c < N; c++) {
		float4 wa = *(const float4 *)(tab[c] + off), wb = *(const float4 *)(tab[c] + off + 4);
		float w[8] = { wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w };
#pragma unroll
		for (int x = 0; x < NT; x++) {
			if (UNI) {
				float a1 = FM(w[x], t[x]);
				a2[c] = FA(a2[c], FM(a0[x], a1));
				a3[c] = FA(a3[c], FM(a1, a1));
			} else qs_term(d[x], nad[x], w[x], Rs[c], a2[c], a3[c]);
		}
		prep(c);
	}
}

/* expands pixels [c*8/N, (c+1)*8/N) (rounded so that the N slices cover 0..7) of word w */
template <int N>
__device__ __forceinline__ void qs_prep_slice(uint2 w, float *f, int c) {
#pragma unroll
	for (int j = 0; j < 8; j++) if (j * N / 8 == c) f[j] = qs_px8(w, j);
}

/* The four sections below are software pipelined by hand: the packed pixel words of the
 * NEXT row are loaded before the current row's ~28*N FP instructions, expanded in slices
 * between the coefficients and differenced afterwards, so neither the LDS latency nor the
 * PRMT->FADD chain sits in front of the FP work. */

/* unroll factors of the row loops of the sections.  Measurement knobs: unrolling by 2 removes 2-4 %
 * of a loop's instructions (address arithmetic, the fp = fn copies) but was measured slower for
 * each loop and for all three: the loop bodies (260-310 instructions at N = 4) stop fitting the
 * instruction cache the four lock-step warps share.  Not re-timed on an H100. */
#ifndef QS_UNROLL_H
#define QS_UNROLL_H 1
#endif
#ifndef QS_UNROLL_B
#define QS_UNROLL_B 1
#endif
#ifndef QS_UNROLL_V
#define QS_UNROLL_V 1
#endif
#define QS_PRAGMA_(x) _Pragma(#x)
#define QS_PRAGMA(x) QS_PRAGMA_(x)

/* horizontal pairs, quantsmooth.h:1527 */
template <int N, bool UNI>
__device__ __forceinline__ void qs_sec_h(const uint2 *pw, const float *const *tab, const float *Rs,
		float *a2, float *a3) {
	float d[8];
	{
		float f[8];
		qs_unpack8(pw[0], f);
#pragma unroll
		for (int x = 0; x < 7; x++) d[x] = FS(f[x], f[x + 1]);
	}
QS_PRAGMA(unroll QS_UNROLL_H)
	for (int y = 0; y < 8; y++) {
		uint2 wn = pw[((y + 1) & 7) * 32];              /* next row (wraps on the last pass) */
		float f[8];
		qs_terms_row<N, 7, UNI>(d, tab, y * 8, Rs, a2, a3, [&](int c) { qs_prep_slice<N>(wn, f, c); });
#pragma unroll
		for (int x = 0; x < 7; x++) d[x] = FS(f[x], f[x + 1]);
	}
}

/* top, bottom, left, right border pairs, quantsmooth.h:1529-1530:
 * (row 0, above), (row 7, below), (column 0, left), (column 7, right) */
template <int N, bool UNI>
__device__ __forceinline__ void qs_sec_border(const uint2 *pw, const float *const *tab, const float *Rs,
		float *a2, float *a3) {
	float d[8];
	{
		float fa[8], fb[8];
		qs_unpack8(pw[0], fa); qs_unpack8(pw[10 * 32], fb);
#pragma unroll
		for (int x = 0; x < 8; x++) d[x] = FS(fa[x], fb[x]);
	}
QS_PRAGMA(unroll QS_UNROLL_B)
	for (int s = 0; s < 4; s++) {
		int sn = (s + 1) & 3;
		int wi = sn == 0 ? 0 : sn == 1 ? 7 : 6 + sn;     /* word of the block edge for step sn */
		uint2 wa = pw[wi * 32], wb = pw[(10 + sn) * 32];
		float fa[8], fb[8];
		qs_terms_row<N, 8, UNI>(d, tab, 64 + s * 8, Rs, a2, a3,
				[&](int c) { qs_prep_slice<N>(wa, fa, c); qs_prep_slice<N>(wb, fb, c); });
#pragma unroll
		for (int x = 0; x < 8; x++) d[x] = FS(fa[x], fb[x]);
	}
}

/* vertical pairs, quantsmooth.h:1531 */
template <int N, bool UNI>
__device__ __forceinline__ void qs_sec_v(const uint2 *pw, const float *const *tab, const float *Rs,
		float *a2, float *a3) {
	float fp[8], d[8];
	{
		float f0[8];
		qs_unpack8(pw[0], f0); qs_unpack8(pw[32], fp);
#pragma unroll
		for (int x = 0; x < 8; x++) d[x] = FS(f0[x], fp[x]);
	}
QS_PRAGMA(unroll QS_UNROLL_V)
	for (int y = 0; y < 7; y++) {
		uint2 wn = pw[min(y + 2, 7) * 32];
		float fn[8];
		qs_terms_row<N, 8, UNI>(d, tab, 96 + y * 8, Rs, a2, a3, [&](int c) { qs_prep_slice<N>(wn, fn, c); });
#pragma unroll
		for (int x = 0; x < 8; x++) { d[x] = FS(fp[x], fn[x]); fp[x] = fn[x]; }
	}
}

/* diagonal pairs, quantsmooth.h:1533-1540: per (y,x) first "\\" then "/" */
template <int N, bool UNI>
__device__ __forceinline__ void qs_sec_diag(const uint2 *pw, const float *const *tab, const float *Rs,
		float *a2, float *a3) {
	float fp[8], d1[8], d2[8];
	{
		float f0[8];
		qs_unpack8(pw[0], f0); qs_unpack8(pw[32], fp);
#pragma unroll
		for (int x = 0; x < 7; x++) { d1[x] = FS(f0[x], fp[x + 1]); d2[x] = FS(f0[x + 1], fp[x]); }
	}
#pragma unroll 1
	for (int y = 0; y < 7; y++) {
		uint2 wn = pw[min(y + 2, 7) * 32];
		float fn[8], t1[8], t2[8], p1[8], p2[8];
		if (UNI) {
#pragma unroll
			for (int x = 0; x < 7; x++) {
				asm("add.rn.sat.f32 %0, %1, %2;" : "=f"(t1[x]) : "f"(Rs[0]), "f"(-fabsf(d1[x])));
				asm("add.rn.sat.f32 %0, %1, %2;" : "=f"(t2[x]) : "f"(Rs[0]), "f"(-fabsf(d2[x])));
				t1[x] = FM(t1[x], t1[x]); t2[x] = FM(t2[x], t2[x]);
				p1[x] = FM(d1[x], t1[x]); p2[x] = FM(d2[x], t2[x]);
			}
		}
#pragma unroll
		for (int c = 0; c < N; c++) {
			const float *t = tab[c] + 160 + y * 16;
			float4 wa = *(const float4 *)t, wb = *(const float4 *)(t + 4);
			float4 wc = *(const float4 *)(t + 8), wd = *(const float4 *)(t + 12);
			float w1[8] = { wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w };
			float w2[8] = { wc.x, wc.y, wc.z, wc.w, wd.x, wd.y, wd.z, wd.w };
#pragma unroll
			for (int x = 0; x < 7; x++) {
				if (UNI) {
					float a1 = FM(w1[x], t1[x]);
					a2[c] = FA(a2[c], FM(p1[x], a1)); a3[c] = FA(a3[c], FM(a1, a1));
					a1 = FM(w2[x], t2[x]);
					a2[c] = FA(a2[c], FM(p2[x], a1)); a3[c] = FA(a3[c], FM(a1, a1));
				} else {
					qs_term(d1[x], -fabsf(d1[x]), w1[x], Rs[c], a2[c], a3[c]);
					qs_term(d2[x], -fabsf(d2[x]), w2[x], Rs[c], a2[c], a3[c]);
				}
			}
			qs_prep_slice<N>(wn, fn, c);
		}
#pragma unroll
		for (int x = 0; x < 7; x++) { d1[x] = FS(fp[x], fn[x + 1]); d2[x] = FS(fp[x + 1], fn[x]); }
#pragma unroll
		for (int x = 0; x < 8; x++) fp[x] = fn[x];
	}
}

/* Lock-step execution: the 4 warps that share an SM sub-partition (warp id % 4) run the same
 * code region at the same time, separated by a named barrier, so that the sub-partition's
 * L0 instruction cache holds ONE unrolled loop body instead of four (free-running warps stalled
 * on instruction fetch). */
/* SYNC encodes (level, warps per sub-partition, lock-step groups per sub-partition):
 * SYNC = level + 16 * WPS + 256 * GS; level 0 = free-running, 1 = barrier per section,
 * 2 = barrier per chunk only.  With GS > 1 a sub-partition hosts GS independent groups that
 * drift against each other, so the ALU-heavy refresh of one overlaps the FMA-heavy sums of
 * the other while the L0 instruction cache still only sees GS loop bodies. */
#define QS_SYNC(level, wps, gs) ((level) + 16 * (wps) + 256 * (gs))
#define QS_SYNC_LEVEL(s) ((s) & 15)
#define QS_SYNC_WPS(s) (((s) >> 4) & 15)
#define QS_SYNC_GS(s) (((s) >> 8) & 15)
template <int SYNC>
__device__ __forceinline__ void qs_group_sync(int grp) {
	/* grp = barrier id | (participating threads << 8), see qs_smooth_kernel */
	if (QS_SYNC_LEVEL(SYNC)) asm volatile("bar.sync %0, %1;" :: "r"(grp & 255), "r"(grp >> 8) : "memory");
}
template <int SYNC>
__device__ __forceinline__ void qs_section_sync(int grp) {
	if (QS_SYNC_LEVEL(SYNC) == 1) qs_group_sync<SYNC>(grp);
}

/* division, rounding and clamped update of the N coefficients of a chunk, quantsmooth.h:1548-1564.
 * Written without control flow (the reference's `if (r)` becomes a select, and the store is
 * unconditional) so that the N dependent chains - divide, round, quant constants, exact
 * division, clamp - interleave; in lock step nothing else could hide their latencies.
 * It also keeps the two sums of the rebalance step (quantsmooth.h:1823-1832: m0 = sum coef*a0,
 * m1 = sum a0*a0 over the AC coefficients) up to date: every AC coefficient passes through here
 * exactly once per iteration, its new value stays inside the quantization interval of a0 (that
 * is what the clamp does), so a0 - already at hand - is also the a0 the rebalance step would
 * recompute from the final value.  The sums live in shared memory (msum[0] = m0, msum[32] = m1).
 */
template <int N>
__device__ __forceinline__ void qs_coef_update(const float *a2s, const float *a3, const uint8_t *idx,
		const QsQuantDev *__restrict__ qd, uint16_t *cs, long long *msum) {
	int q[N], c[N], r[N]; uint32_t m31[N]; uint16_t *slot[N];
	long long m0 = msum[0], m1 = msum[32];
#pragma unroll
	for (int k = 0; k < N; k++) {
		int i = idx[k];
		slot[k] = cs + (i >> 1) * 64 + (i & 1);
		q[k] = __ldg(&qd->q[i]); m31[k] = __ldg(&qd->m31[i]);
		c[k] = (short)*slot[k];
	}
#pragma unroll
	for (int k = 0; k < N; k++) {
		float qv = FM(__fdiv_rn(a2s[k], a3[k]), 35184372088832.0f);     /* * 2^45, exact */
		r[k] = qs_cvtt_x86(roundf(qv));
	}
#pragma unroll
	for (int k = 0; k < N; k++) {
		int a0 = qs_orig_coef(c[k], q[k], m31[k]);
		int d0 = (q[k] - 1) >> 1, d1 = q[k] >> 1;
		int dh = a0 + (a0 < 0 ? d1 : d0), dl = a0 - (a0 > 0 ? d1 : d0);
		int add = (int)((unsigned)c[k] - (unsigned)r[k]);
		add = min(add, dh); add = max(add, dl);
		add = r[k] ? add : c[k];
		*slot[k] = (uint16_t)add;
		m0 += add * a0; m1 += a0 * a0;
	}
	msum[0] = m0; msum[32] = m1;
}

template <int N, bool DIAG, int SYNC, bool UNI>
__device__ __forceinline__ void qs_chunk_full(const QsChunk &ch, const float *tabs, const uint2 *pw,
		const QsQuantDev *__restrict__ qd, uint16_t *cs, int grp, QsPh &ph, const uint32_t *nh, uint32_t *h, long long *msum) {
	const float *tab[N]; float Rs[N], a2[N], a3[N];
	const int TS = DIAG ? QS_TAB_DIAG : QS_TAB_PLAIN;
#pragma unroll
	for (int c = 0; c < N; c++) {
		int i = ch.idx[c];
		tab[c] = tabs + i * TS; Rs[c] = __ldg(&qd->Rs[i]); a2[c] = 0.0f; a3[c] = 0.0f;
	}
	QS_PH_MARK(ph, 4);
	qs_sec_h<N, UNI>(pw, tab, Rs, a2, a3);
	qs_section_sync<SYNC>(grp);
	QS_PH_MARK(ph, 5);
	qs_sec_border<N, UNI>(pw, tab, Rs, a2, a3);
	qs_section_sync<SYNC>(grp);
	QS_PH_MARK(ph, 6);
	qs_sec_v<N, UNI>(pw, tab, Rs, a2, a3);
	QS_PH_MARK(ph, 7);
	if (DIAG) { qs_section_sync<SYNC>(grp); qs_sec_diag<N, UNI>(pw, tab, Rs, a2, a3); }
	qs_section_sync<SYNC>(grp);
	QS_PH_MARK(ph, 8);
	/* the next chunk's header travels while the divisions below are in flight */
	h[0] = __ldg(nh); h[1] = __ldg(nh + 1); h[2] = __ldg(nh + 2);
	qs_coef_update<N>(a2, a3, ch.idx, qd, cs, msum);
	QS_PH_MARK(ph, 9);
}

/* the two edge coefficients of an anti-diagonal: idx[0] lies in row 0 (i <= 7: no vertical
 * terms), idx[1] in column 0 (i & 7 == 0: no horizontal terms) */
template <bool DIAG, int SYNC>
__device__ __forceinline__ void qs_chunk_edge(const QsChunk &ch, const float *tabs, const uint2 *pw,
		const QsQuantDev *__restrict__ qd, uint16_t *cs, int grp, QsPh &ph, const uint32_t *nh, uint32_t *h, long long *msum) {
	const float *tab[2]; float Rs[2], a2[2], a3[2];
	const int TS = DIAG ? QS_TAB_DIAG : QS_TAB_PLAIN;
#pragma unroll
	for (int c = 0; c < 2; c++) {
		int i = ch.idx[c];
		tab[c] = tabs + i * TS; Rs[c] = __ldg(&qd->Rs[i]); a2[c] = 0.0f; a3[c] = 0.0f;
	}
	QS_PH_MARK(ph, 4);
	qs_sec_h<1, false>(pw, tab, Rs, a2, a3);
	qs_section_sync<SYNC>(grp);
	QS_PH_MARK(ph, 5);
	qs_sec_border<2, false>(pw, tab, Rs, a2, a3);
	qs_section_sync<SYNC>(grp);
	QS_PH_MARK(ph, 6);
	qs_sec_v<1, false>(pw, tab + 1, Rs + 1, a2 + 1, a3 + 1);
	QS_PH_MARK(ph, 7);
	if (DIAG) { qs_section_sync<SYNC>(grp); qs_sec_diag<2, false>(pw, tab, Rs, a2, a3); }
	qs_section_sync<SYNC>(grp);
	QS_PH_MARK(ph, 8);
	h[0] = __ldg(nh); h[1] = __ldg(nh + 1); h[2] = __ldg(nh + 2);
	qs_coef_update<2>(a2, a3, ch.idx, qd, cs, msum);
	QS_PH_MARK(ph, 9);
}

/* "mixed" chunk (schedule type 3): NF (1 or 2) full coefficients of an anti-diagonal together with
 * its two edge coefficients - idx[NF] lies in row 0 (no vertical terms), idx[NF+1] in column 0
 * (no horizontal terms; quantsmooth.h:1527, 1531).  The edge coefficients share the pixel
 * expansion, the differences and the table-load slots of the full ones instead of paying for
 * single-coefficient horizontal / vertical passes of their own, and the diagonal has one chunk
 * (one barrier, one header, one update batch) less. */
template <int NF, bool DIAG, int SYNC>
__device__ __forceinline__ void qs_chunk_mixed(const QsChunk &ch, const float *tabs, const uint2 *pw,
		const QsQuantDev *__restrict__ qd, uint16_t *cs, int grp, QsPh &ph, const uint32_t *nh, uint32_t *h, long long *msum) {
	const int NT = NF + 2, TS = DIAG ? QS_TAB_DIAG : QS_TAB_PLAIN;
	const float *tab[NT]; float Rs[NT], a2[NT], a3[NT];
#pragma unroll
	for (int c = 0; c < NT; c++) {
		int i = ch.idx[c];
		tab[c] = tabs + i * TS; Rs[c] = __ldg(&qd->Rs[i]); a2[c] = 0.0f; a3[c] = 0.0f;
	}
	QS_PH_MARK(ph, 4);
	qs_sec_h<NF + 1, false>(pw, tab, Rs, a2, a3);           /* full coefficients + the row-0 one */
	qs_section_sync<SYNC>(grp);
	QS_PH_MARK(ph, 5);
	qs_sec_border<NT, false>(pw, tab, Rs, a2, a3);
	qs_section_sync<SYNC>(grp);
	QS_PH_MARK(ph, 6);
	{                                                       /* full coefficients + the column-0 one */
		const float *tv[NF + 1]; float Rv[NF + 1], v2[NF + 1], v3[NF + 1];
#pragma unroll
		for (int c = 0; c < NF; c++) { tv[c] = tab[c]; Rv[c] = Rs[c]; v2[c] = a2[c]; v3[c] = a3[c]; }
		tv[NF] = tab[NF + 1]; Rv[NF] = Rs[NF + 1]; v2[NF] = a2[NF + 1]; v3[NF] = a3[NF + 1];
		qs_sec_v<NF + 1, false>(pw, tv, Rv, v2, v3);
#pragma unroll
		for (int c = 0; c < NF; c++) { a2[c] = v2[c]; a3[c] = v3[c]; }
		a2[NF + 1] = v2[NF]; a3[NF + 1] = v3[NF];
	}
	QS_PH_MARK(ph, 7);
	if (DIAG) { qs_section_sync<SYNC>(grp); qs_sec_diag<NT, false>(pw, tab, Rs, a2, a3); }
	qs_section_sync<SYNC>(grp);
	QS_PH_MARK(ph, 8);
	h[0] = __ldg(nh); h[1] = __ldg(nh + 1); h[2] = __ldg(nh + 2);
	qs_coef_update<NT>(a2, a3, ch.idx, qd, cs, msum);
	QS_PH_MARK(ph, 9);
}


/* IDCT of the lane's block from shared coefficients into the shared pixel words */
__device__ __forceinline__ void qs_refresh(const uint32_t *cw, uint2 *pw) {
	int ws[64];
#pragma unroll
	for (int xp = 0; xp < 4; xp++) {
		int a[8], b[8], oa[8], ob[8];
#pragma unroll
		for (int k = 0; k < 8; k++) {
			uint32_t w = cw[(k * 4 + xp) * 32];
			a[k] = (short)(w & 0xffff); b[k] = (int)w >> 16;
		}
		qs_islow_1d<1024>(a, oa); qs_islow_1d<1024>(b, ob);
#pragma unroll
		for (int k = 0; k < 8; k++) {
			ws[k * 8 + 2 * xp] = oa[k] >> 11;
			ws[k * 8 + 2 * xp + 1] = ob[k] >> 11;
		}
	}
	uint32_t lo[8], hi[8];
	qs_islow_rows(ws, lo, hi);
#pragma unroll
	for (int y = 0; y < 8; y++) pw[y * 32] = make_uint2(lo[y], hi[y]);
	pw[8 * 32] = qs_gather_col(lo, 0);
	pw[9 * 32] = qs_gather_col(hi, 3);
}

/* fdct_clamp, quantsmooth.h:343-347, 551-561: FDCT, round half away, clamp every
 * coefficient (DC included) into the quantization interval of its current value */
__device__ __forceinline__ void qs_fdct_clamp(float *f, const QsQuantDev *__restrict__ qd, uint16_t *cs) {
	qs_fdct_8x8(f);
#pragma unroll
	for (int x = 0; x < 64; x++) {
		uint16_t *slot = cs + (x >> 1) * 64 + (x & 1);
		int c = (short)*slot;
		int q = __ldg(&qd->q[x]);
		int a0 = qs_orig_coef(c, q, __ldg(&qd->m31[x]));
		int d0 = (q - 1) >> 1, d1 = q >> 1;
		int dh = a0 + (a0 < 0 ? d1 : d0), dl = a0 - (a0 > 0 ? d1 : d0);
		int add = qs_cvtt_x86(roundf(f[x]));
		add = min(add, dh); add = max(add, dl);
		*slot = (uint16_t)add;
	}
}

/* the same for the LOW_QUALITY kernel: the transformed block is parked in shared memory
 * (fs[k * 32]) and the clamp loop is rolled - that kernel's top stall was instruction fetch -
 * and, like qs_coef_update, it leaves the two sums of the rebalance step
 * (m0 = sum coef*a0, m1 = sum a0*a0 over the AC coefficients; the clamp keeps the new value in
 * the quantization interval of a0, so a0 is what the rebalance step would recompute) */
__device__ __forceinline__ void qs_fdct_clamp_rolled(float *f, float *fs, const QsQuantDev *__restrict__ qd, uint16_t *cs,
		long long &m0, long long &m1) {
	qs_fdct_8x8(f);
#pragma unroll
	for (int x = 0; x < 64; x++) fs[x * 32] = f[x];
	long long s0 = 0, s1 = 0;
#pragma unroll 8
	for (int x = 0; x < 64; x++) {
		uint16_t *slot = cs + (x >> 1) * 64 + (x & 1);
		int c = (short)*slot;
		int q = __ldg(&qd->q[x]);
		int a0 = qs_orig_coef(c, q, __ldg(&qd->m31[x]));
		int d0 = (q - 1) >> 1, d1 = q >> 1;
		int dh = a0 + (a0 < 0 ? d1 : d0), dl = a0 - (a0 > 0 ? d1 : d0);
		int add = qs_cvtt_x86(roundf(fs[x * 32]));
		add = min(add, dh); add = max(add, dl);
		*slot = (uint16_t)add;
		if (x) { s0 += add * a0; s1 += a0 * a0; }
	}
	m0 = s0; m1 = s1;
}

/* JOINT_YUV chroma predictor + fdct_clamp, quantsmooth.h:577-579, 894-921, 551-561 */
__device__ __noinline__ void qs_joint_predict(const uint8_t *__restrict__ img, const uint8_t *__restrict__ img2,
		int stride, const QsQuantDev *__restrict__ qd, uint16_t *cs) {
	float f[64];
#pragma unroll
	for (int y = 0; y < 8; y++) {
#pragma unroll
		for (int x = 0; x < 8; x++) {
			int sA, sB;
			const uint8_t *A = img2 + y * stride + x, *B = img + y * stride + x;
			float scale = qs_regress(A, B, stride, sA, sB);
			float a = FM(FA(FM((float)((int)A[0] * 16 - sA), scale), (float)sB), 1.0f / 16);
			a = FS(a < 0 ? 0.0f : a, 128.0f);
			f[y * 8 + x] = a > 128.0f ? 128.0f : a;
		}
	}
	qs_fdct_clamp(f, qd, cs);
}

/* rebalance, quantsmooth.h:1566-1568, 1823-1848: the two sums over the AC coefficients ... */
__device__ __forceinline__ void qs_rebalance_sums(const QsQuantDev *__restrict__ qd, const uint16_t *cs, long long &m0, long long &m1) {
	long long s0 = 0, s1 = 0;
	/* 63 independent iterations, latency bound when rolled (LDS -> LDG -> IMAD.HI); unrolled
	 * by 7 the loads of seven coefficients are in flight together */
#pragma unroll 7
	for (int k = 1; k < 64; k++) {
		int c = (short)cs[(k >> 1) * 64 + (k & 1)];
		int a0 = qs_orig_coef(c, __ldg(&qd->q[k]), __ldg(&qd->m31[k]));
		s0 += c * a0; s1 += a0 * a0;
	}
	m0 = s0; m1 = s1;
}
/* ... and the rescaling they decide (the smoothing kernel and the LOW_QUALITY kernel keep the
 * sums up to date while they clamp, qs_coef_update / qs_fdct_clamp_rolled) */
__device__ __forceinline__ void qs_rebalance(const QsQuantDev *__restrict__ qd, uint16_t *cs, long long m0, long long m1) {
	if (m1 > m0 && m0 != 0) {
		int mul = (int)(((m1 << 13) + (m0 >> 1)) / m0);
#pragma unroll 7
		for (int k = 1; k < 64; k++) {
			uint16_t *slot = cs + (k >> 1) * 64 + (k & 1);
			int c = (short)*slot;
			int q = __ldg(&qd->q[k]);
			int a0 = qs_orig_coef(c, q, __ldg(&qd->m31[k]));
			int d0 = (q - 1) >> 1, d1 = q >> 1;
			int dh = a0 + (a0 < 0 ? d1 : d0), dl = a0 - (a0 > 0 ? d1 : d0);
			int add = (int)((unsigned)c * (unsigned)mul + 0x1000u) >> 13;
			add = min(add, dh); add = max(add, dl);
			*slot = (uint16_t)add;
		}
	}
}

template <bool DIAG, int SYNC>
__global__ void __launch_bounds__(QS_SYNC_WPS(SYNC) * 128, 1) qs_smooth_kernel(const QsJob *__restrict__ jobs,
		int njobs, int total_tiles, const float *__restrict__ tables_g, int *__restrict__ tile_counter,
		int flags, int clamp_out, const int *__restrict__ bad) {
	extern __shared__ __align__(16) uint32_t smem[];
	__shared__ int s_tile[16], s_next[16];
	__shared__ int s_sig[32];
	const int TS = DIAG ? QS_TAB_DIAG : QS_TAB_PLAIN;
	const int tab_words = 64 * TS;
	float *tabs = (float *)smem;
	{
		/* Stage the weight tables (40-80 KB) with one TMA bulk copy (cp.async.bulk, UBLKCP in
		 * SASS) completing on an mbarrier: the persistent CTA does this once, all 16 warps
		 * wait on phase 0. */
		__shared__ __align__(8) unsigned long long tab_bar;
		uint32_t bar = (uint32_t)__cvta_generic_to_shared(&tab_bar);
		uint32_t dst = (uint32_t)__cvta_generic_to_shared(tabs);
		uint32_t bytes = (uint32_t)tab_words * 4;
		if (threadIdx.x == 0) {
			asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar) : "memory");
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
		}
		__syncthreads();
		if (threadIdx.x == 0) {
			asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
			asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
					:: "r"(dst), "l"(tables_g), "r"(bytes), "r"(bar) : "memory");
		}
		asm volatile("{\n\t.reg .pred p;\n\tQS_TAB_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t"
				"@!p bra QS_TAB_WAIT;\n\t}" :: "r"(bar) : "memory");
	}
	int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int NG = 4 * QS_SYNC_GS(SYNC);                /* lock-step groups in this CTA */
	const int WPG = QS_SYNC_WPS(SYNC) / QS_SYNC_GS(SYNC);   /* warps per group, all on one sub-partition */
	int grp = warp % NG, wig = warp / NG;
	uint32_t *wbase = smem + tab_words + warp * QS_WARP_WORDS;
	uint32_t *cw = wbase + lane;                        /* coefficient pair p at cw[p * 32] */
	uint16_t *cs = (uint16_t *)wbase + lane * 2;        /* coefficient i at cs[(i>>1)*64 + (i&1)] */
	uint2 *pw = (uint2 *)(wbase + 32 * 32) + lane;      /* pixel word j at pw[j * 32] */
	long long *msum = (long long *)(wbase + QS_WARP_MSUM) + lane;   /* rebalance sums: msum[0], msum[32] */

	/* Tile schedule of the lock-step groups: first `a_tiles` group tiles of WPG warp tiles
	 * each (dynamic, one atomic per group tile); then the left-over warp tiles are spread
	 * evenly over ALL groups (0..WPG warps active per group, static) so that the last wave is
	 * short instead of leaving most sub-partitions idle for a whole tile time. */
	const int G = gridDim.x * NG;
	const int a_tiles = (total_tiles / (WPG * G)) * G;
	const int left = total_tiles - a_tiles * WPG, lbase = left / G, lextra = left - lbase * G;
	int gbar = (1 + grp) | ((WPG * 32) << 8);           /* barrier id | participating threads */
	bool last = false;
	QsPh ph;
#ifdef QS_PHASE_CLOCKS
	__shared__ uint32_t s_ph[32][QS_NPHASE];
	for (int k = lane; k < QS_NPHASE; k += 32) s_ph[warp][k] = 0;
	__syncwarp();
	ph.start(s_ph[warp]);
#endif

	/* The group tile after the current one is known one tile ahead (its atomic ran during the
	 * previous tile), so the group can ask L2 for its coefficients and pixel rows while it still
	 * works on the current tile: the prologue's DRAM round trips leave the critical path. */
	if (QS_SYNC_LEVEL(SYNC) && wig == 0 && lane == 0) {
		s_tile[grp] = atomicAdd(tile_counter, 1);
		s_next[grp] = atomicAdd(tile_counter, 1);
	}
	for (;;) {
		int tile = 0, gnext = 0, gnext2 = 0;
		if (QS_SYNC_LEVEL(SYNC)) {
			if (last) break;
			qs_group_sync<SYNC>(gbar);
			int gt = *(volatile int *)&s_tile[grp];
			gnext = *(volatile int *)&s_next[grp];
			qs_group_sync<SYNC>(gbar);                  /* s_tile / s_next may be rewritten from here on */
			if (wig == 0 && lane == 0) gnext2 = atomicAdd(tile_counter, 1);    /* consumed at the end of this tile */
			if (gt < a_tiles) tile = gt * WPG + wig;
			else {
				int j = blockIdx.x * NG + grp;          /* this group's left-over share */
				int nw = lbase + (j < lextra ? 1 : 0);
				if (wig >= nw) break;                   /* idle warps leave; the rest re-size the barrier */
				tile = a_tiles * WPG + j * lbase + min(j, lextra) + wig;
				gbar = (1 + grp) | ((nw * 32) << 8);
				last = true;
			}
		} else {
			if (lane == 0) tile = atomicAdd(tile_counter, 1);
			tile = __shfl_sync(0xffffffffu, tile, 0);
			if (tile >= total_tiles) break;
		}
		const int gsync = gbar;
		const bool active = true;
		QS_PH_MARK(ph, 0);
		const QsJob *job = jobs + qs_find_job(jobs, njobs, tile);
		int nblocks = job->nblocks;
		int b = (tile - job->tile_begin) * 32 + lane;
		/* a stopped component walks through the passes like any other (the barrier sequence of
		 * its lock-step group must not change) but never writes anything back */
		bool valid = active && b < nblocks && !qs_job_state(job, bad);
		if (b >= nblocks) b = nblocks - 1;              /* idle lanes shadow the last block */
		int W = job->wblk, stride = job->stride;
		int by = b / W, bx = b - by * W;
		int16_t *cptr = job->coef + (size_t)b * 64;
		const QsQuantDev *qd = job->quant;
		const uint8_t *img = job->plane + (size_t)(by * 8 + 1) * stride + QS_PLANE_PAD + bx * 8;

		{
			const int4 *p = (const int4 *)cptr;
#pragma unroll
			for (int j = 0; j < 8; j++) {
				int4 v = p[j];
				cw[(j * 4 + 0) * 32] = v.x; cw[(j * 4 + 1) * 32] = v.y;
				cw[(j * 4 + 2) * 32] = v.z; cw[(j * 4 + 3) * 32] = v.w;
			}
		}
		if (job->plane2) {
			const uint8_t *img2 = job->plane2 + (size_t)(by * 8 + 1) * stride + QS_PLANE_PAD + bx * 8;
			qs_joint_predict(img, img2, stride, qd, cs);
		}
		{                                               /* border, quantsmooth.h:1396-1401 */
			pw[10 * 32] = *(const uint2 *)(img - stride);
			pw[11 * 32] = *(const uint2 *)(img + (size_t)8 * stride);
			uint32_t l0 = 0, l1 = 0, r0 = 0, r1 = 0;
#pragma unroll
			for (int y = 0; y < 4; y++) {
				l0 |= (uint32_t)img[(size_t)y * stride - 1] << (8 * y);
				l1 |= (uint32_t)img[(size_t)(y + 4) * stride - 1] << (8 * y);
				r0 |= (uint32_t)img[(size_t)y * stride + 8] << (8 * y);
				r1 |= (uint32_t)img[(size_t)(y + 4) * stride + 8] << (8 * y);
			}
			pw[12 * 32] = make_uint2(l0, l1);
			pw[13 * 32] = make_uint2(r0, r1);
		}
		/* The first refresh of a block would re-render exactly what the IDCT pass just wrote to
		 * the plane (same coefficients, deterministic IDCT), so those 64 pixels are loaded
		 * instead of computed - unless the JOINT_YUV predictor changed the coefficients. */
		msum[0] = 0; msum[32] = 0;
		if (QS_SYNC_LEVEL(SYNC) && gnext < a_tiles) {
			/* next group tile, if it lies in the same component: one coefficient line per lane
			 * (32 blocks x 128 B), the ten pixel rows the prologue reads (3 lines each) */
			int nb0 = ((gnext * WPG + wig) - job->tile_begin) * 32;
			if (nb0 >= 0 && nb0 + 32 <= nblocks) {
				asm volatile("prefetch.global.L2 [%0];" :: "l"(job->coef + ((size_t)nb0 + lane) * 64));
				int nby = nb0 / W, nbx = nb0 - nby * W;
				if (lane < 30 && nbx * 8 + (lane % 3) * 128 < W * 8) {          /* stay inside the row */
					const uint8_t *np = job->plane + (size_t)(nby * 8 + lane / 3) * stride + QS_PLANE_PAD + nbx * 8 + (lane % 3) * 128;
					asm volatile("prefetch.global.L2 [%0];" :: "l"(np));
				}
			}
		}
		const bool fresh_px = job->plane2 == NULL;
		/* Warps of a lock-step group may sit in different components (a group tile or the
		 * balanced tail can straddle jobs).  Their barrier sequences must be identical, so a
		 * mixed group takes the table-independent schedule and always refreshes at chunk 0. */
		bool mixed = false;
		if (QS_SYNC_LEVEL(SYNC)) {
			int sig = __ldg(&qd->sched_slot) * 2 + (fresh_px ? 1 : 0);
			if (lane == 0) s_sig[warp] = sig;
			qs_group_sync<SYNC>(gsync);
			int nw = (gsync >> 8) >> 5;
			for (int k = 0; k < nw; k++) mixed = mixed || *(volatile int *)&s_sig[k * NG + grp] != sig;
			mixed = __any_sync(0xffffffffu, mixed);
		}
		const bool skip0 = fresh_px && !mixed;
		if (fresh_px) {
			uint32_t lo[8], hi[8];
#pragma unroll
			for (int y = 0; y < 8; y++) {
				uint2 v = *(const uint2 *)(img + (size_t)y * stride);
				lo[y] = v.x; hi[y] = v.y; pw[y * 32] = v;
			}
			pw[8 * 32] = qs_gather_col(lo, 0);
			pw[9 * 32] = qs_gather_col(hi, 3);
		}
		QS_PH_MARK(ph, 1);

		int nch = mixed ? d_nchunks : __ldg(&qd->nchunks);
		/* 12-byte chunk headers (type, n, first, -, idx[8]); warp-uniform.  Each chunk fetches its
		 * successor's header before its own divisions, so no chunk starts with a load latency. */
		const uint32_t *cp = (const uint32_t *)(mixed ? d_chunks : qd->chunks);
		uint32_t h[3] = { __ldg(cp), __ldg(cp + 1), __ldg(cp + 2) };
#pragma unroll 1
		for (int ci = 0; ci < nch; ci++) {
			QsChunk ch;
			ch.type = h[0] & 255; ch.n = (h[0] >> 8) & 255; ch.first = (h[0] >> 16) & 255; ch.pad = 0;
			ch.idx[0] = h[1] & 255; ch.idx[1] = (h[1] >> 8) & 255; ch.idx[2] = (h[1] >> 16) & 255; ch.idx[3] = h[1] >> 24;
			ch.idx[4] = h[2] & 255; ch.idx[5] = (h[2] >> 8) & 255; ch.idx[6] = (h[2] >> 16) & 255; ch.idx[7] = h[2] >> 24;
			const uint32_t *nh = cp + 3 * min(ci + 1, nch - 1);
			qs_group_sync<SYNC>(gsync);
			QS_PH_MARK(ph, 2);
			/* the reference re-renders only if a coefficient changed (need_refresh); an
			 * unconditional refresh at each anti-diagonal start is value-identical */
			if (ch.first && !(ci == 0 && skip0)) { qs_refresh(cw, pw); qs_group_sync<SYNC>(gsync); }
			QS_PH_MARK(ph, 3);
			if (ch.type == 1) qs_chunk_edge<DIAG, SYNC>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
			else if (ch.type == 3) {
				if (ch.n == 2) qs_chunk_mixed<2, DIAG, SYNC>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
				else qs_chunk_mixed<1, DIAG, SYNC>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
			}
			else if (ch.type == 2) {
				if (ch.n == 4) qs_chunk_full<4, DIAG, SYNC, true>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
				else if (ch.n == 3) qs_chunk_full<3, DIAG, SYNC, true>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
				else qs_chunk_full<2, DIAG, SYNC, true>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
			}
			else if (ch.n == 4) qs_chunk_full<4, DIAG, SYNC, false>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
			else if (ch.n == 3) qs_chunk_full<3, DIAG, SYNC, false>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
			else if (ch.n == 2) qs_chunk_full<2, DIAG, SYNC, false>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
			else qs_chunk_full<1, DIAG, SYNC, false>(ch, tabs, pw, qd, cs, gsync, ph, nh, h, msum);
		}
		QS_PH_MARK(ph, 10);

		if (!(flags & QS_NO_REBALANCE) && !(!job->luma && (flags & QS_NO_REBALANCE_UV)))
			qs_rebalance(qd, cs, msum[0], msum[32]);
		QS_PH_MARK(ph, 11);

		if (valid) {
			int4 *p = (int4 *)cptr;
#pragma unroll
			for (int j = 0; j < 8; j++) {
				uint32_t w[4];
#pragma unroll
				for (int k = 0; k < 4; k++) {
					w[k] = cw[(j * 4 + k) * 32];
					if (clamp_out) {                    /* quantsmooth.h:2670-2689 */
						int a = (short)(w[k] & 0xffff), c2 = (int)w[k] >> 16;
						a = min(max(a, -1023), 1023); c2 = min(max(c2, -1023), 1023);
						w[k] = (uint32_t)(a & 0xffff) | ((uint32_t)c2 << 16);
					}
				}
				p[j] = make_int4((int)w[0], (int)w[1], (int)w[2], (int)w[3]);
			}
		}
		__syncwarp();
		if (QS_SYNC_LEVEL(SYNC) && wig == 0 && lane == 0) { s_tile[grp] = gnext; s_next[grp] = gnext2; }
		QS_PH_MARK(ph, 12);
	}
#ifdef QS_PHASE_CLOCKS
	__syncwarp();
	if (lane < QS_NPHASE) atomicAdd(&qs_phase_acc[lane], (unsigned long long)s_ph[warp][lane]);
#endif
}

#ifdef QS_PHASE_CLOCKS
extern "C" int qs_read_phase_clocks(unsigned long long *out, int reset) {
	unsigned long long z[QS_NPHASE] = { 0 };
	if (cudaMemcpyFromSymbol(out, qs_phase_acc, sizeof(z)) != cudaSuccess) return -1;
	if (reset && cudaMemcpyToSymbol(qs_phase_acc, z, sizeof(z)) != cudaSuccess) return -1;
	return QS_NPHASE;
}
#endif

/* ------------------------------------------------------------------------------------------
 * LOW_QUALITY (q0-2) block function, quantsmooth.h:924-938 + 1162-1178 (scalar branch, which
 * truncates `a -= a0/an` to int - the reference's SIMD branches keep it in float and give
 * different results; the scalar build is the contract).  One thread per block, no tables:
 * range from the coefficient magnitudes, 8-neighbour one-shot filter, FDCT + clamp,
 * rebalance.  ~10 k instructions and ~420 B of traffic per block: the HBM-bound mode.
 * ------------------------------------------------------------------------------------------ */
__device__ __forceinline__ void qs_lowq_row(const uint8_t *__restrict__ p, float *r) {
	/* 10 pixels x = -1..8 of one plane row as 1 + px * 2^-15 (qs_px); p points at x = 0 (8-byte aligned) */
	uint2 w = *(const uint2 *)p;
	r[0] = qs_px((uint32_t)p[-1], 0); r[9] = qs_px((uint32_t)p[8], 0);
#pragma unroll
	for (int k = 0; k < 4; k++) { r[1 + k] = qs_px(w.x, k); r[5 + k] = qs_px(w.y, k); }
}

#ifndef QS_LOWQ_MINB
#define QS_LOWQ_MINB 4
#endif
__global__ void __launch_bounds__(128, QS_LOWQ_MINB) qs_lowq_kernel(const QsJob *__restrict__ jobs, int njobs, int total_tiles,
		int flags, int clamp_out, const int *__restrict__ bad) {
	__shared__ uint32_t sm[4 * 32 * 32];
	__shared__ float sf[4 * 64 * 32];
	int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	int tile = blockIdx.x * 4 + warp;
	if (tile >= total_tiles) return;
	const QsJob *job = jobs + qs_find_job(jobs, njobs, tile);
	int b = (tile - job->tile_begin) * 32 + lane;
	if (b >= job->nblocks || qs_job_state(job, bad)) return;
	uint32_t *cw = sm + warp * 1024 + lane;
	uint16_t *cs = (uint16_t *)(sm + warp * 1024) + lane * 2;
	int W = job->wblk, stride = job->stride;
	int by = b / W, bx = b - by * W;
	int16_t *cptr = job->coef + (size_t)b * 64;
	const QsQuantDev *qd = job->quant;
	const uint8_t *img = job->plane + (size_t)(by * 8 + 1) * stride + QS_PLANE_PAD + bx * 8;
	{
		const int4 *p = (const int4 *)cptr;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			int4 v = p[j];
			cw[(j * 4 + 0) * 32] = v.x; cw[(j * 4 + 1) * 32] = v.y;
			cw[(j * 4 + 2) * 32] = v.z; cw[(j * 4 + 3) * 32] = v.w;
		}
	}
	long long m0 = 0, m1 = 0; bool have_sums = false;
	if (job->plane2) {                                  /* JOINT_YUV predictor, then straight to rebalance (928) */
		const uint8_t *img2 = job->plane2 + (size_t)(by * 8 + 1) * stride + QS_PLANE_PAD + bx * 8;
		qs_joint_predict(img, img2, stride, qd, cs);
	} else {
		float range = 0.0f; int sum = 0;
#pragma unroll 7
		for (int x = 1; x < 64; x++) {
			int a = (short)cs[(x >> 1) * 64 + (x & 1)]; a = a < 0 ? -a : a;
			range = FA(range, (float)((int)__ldg(&qd->q[x]) * a)); sum += a;
		}
		if (sum) range = FM(range, __fdiv_rn(4.0f, (float)sum));
		if (range > 128.0f) range = 128.0f;
		range = roundf(range);
		const float c0 = 2.0f, c1 = FM(2.0f, 0.70710678118654752440f);   /* c0 * sqrtf(0.5f) */
		/* The same exact rescaling as in the smoothing kernel: pixels as 1 + p * 2^-15, so a
		 * difference is d * 2^-15 with no int -> float conversion, and with range * 2^-15 the clamp
		 * max(range - |d|, 0) is one add.sat.  The products carry pure power-of-two factors (2^-75
		 * in a0, 2^-60 in an, no underflow: tools/lowq_scaling_check.c checks every (range, d) and
		 * 2e7 random pixels against the plain form); the quotient comes out scaled by 2^-15. */
		const float rs = FM(range, 3.0517578125e-05f);
		float r0[10], r1[10], r2[10];
		qs_lowq_row(img - stride, r0); qs_lowq_row(img, r1);
		/* rows in a rolled loop (one 8-pixel body instead of 64 pixels of straight-line code),
		 * the filtered pixels parked in shared memory: together with the rolled clamp loop this
		 * keeps the kernel's instruction footprint small */
		float *f = sf + warp * 2048 + lane;
#pragma unroll 1
		for (int y = 0; y < 8; y++) {
			qs_lowq_row(img + (size_t)(y + 1) * stride, r2);
#pragma unroll
			for (int x = 0; x < 8; x++) {
				const float ac = r1[x + 1]; float a0 = 0.0f, an = 0.0f;
#define NB(c_, v_) { float d = FS(ac, v_), t, aw; \
	asm("add.rn.sat.f32 %0, %1, %2;" : "=f"(t) : "f"(rs), "f"(-fabsf(d))); \
	t = FM(t, t); aw = FM(c_, t); a0 = FA(a0, FM(FM(d, t), aw)); an = FA(an, FM(aw, aw)); }
				NB(c1, r0[x]) NB(c0, r0[x + 1]) NB(c1, r0[x + 2])
				NB(c0, r1[x]) NB(c0, r1[x + 2])
				NB(c1, r2[x]) NB(c0, r2[x + 1]) NB(c1, r2[x + 2])
#undef NB
				const float af = FM(FS(ac, 1.0f), 32768.0f);            /* (float)pixel, exact */
				float fv = FS(af, 128.0f);
				if (an > 0.0f) fv = (float)(qs_cvtt_x86(FS(af, FM(__fdiv_rn(a0, an), 32768.0f))) - 128);
				f[(y * 8 + x) * 32] = fv;
			}
#pragma unroll
			for (int k = 0; k < 10; k++) { r0[k] = r1[k]; r1[k] = r2[k]; }
		}
		float fr[64];
#pragma unroll
		for (int k = 0; k < 64; k++) fr[k] = f[k * 32];
		qs_fdct_clamp_rolled(fr, f, qd, cs, m0, m1);
		have_sums = true;
	}
	if (!(flags & QS_NO_REBALANCE) && !(!job->luma && (flags & QS_NO_REBALANCE_UV))) {
		if (!have_sums) qs_rebalance_sums(qd, cs, m0, m1);
		qs_rebalance(qd, cs, m0, m1);
	}
	{
		int4 *p = (int4 *)cptr;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			uint32_t w[4];
#pragma unroll
			for (int k = 0; k < 4; k++) {
				w[k] = cw[(j * 4 + k) * 32];
				if (clamp_out) {
					int a = (short)(w[k] & 0xffff), c2 = (int)w[k] >> 16;
					a = min(max(a, -1023), 1023); c2 = min(max(c2, -1023), 1023);
					w[k] = (uint32_t)(a & 0xffff) | ((uint32_t)c2 << 16);
				}
			}
			p[j] = make_int4((int)w[0], (int)w[1], (int)w[2], (int)w[3]);
		}
	}
}

/* ------------------------------------------------------------------------------------------
 * dequantize-only / clamp-only fallbacks (quantsmooth.h:2551-2566, 2670-2689)
 * ------------------------------------------------------------------------------------------ */
__global__ void qs_scale_clamp_kernel(int16_t *__restrict__ coef, size_t n, const QsQuantDev *__restrict__ qd,
		int dequant, int clamp) {
	size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	size_t step = (size_t)gridDim.x * blockDim.x;
	for (; i < n; i += step) {
		int c = coef[i];
		if (dequant) c = (short)(c * (int)__ldg(&qd->qraw[i & 63]));
		if (clamp) c = min(max(c, -1023), 1023);
		coef[i] = (int16_t)c;
	}
}

/* ------------------------------------------------------------------------------------------
 * down-sampled luma plane with replicated borders, quantsmooth.h:2753-2815.
 * One thread per output pixel of the PADDED destination plane (incl. borders), so border
 * replication needs no second pass: every thread clamps its source coordinates.
 * src: Y plane (w = W*8, h = H*8 valid pixels).  dst: (w2+2) x (h2+2) with w2/h2 = chroma
 * plane size; valid area w1 x h1 = ceil(w/ws) x ceil(h/hs).
 * ------------------------------------------------------------------------------------------ */
__global__ void qs_downsample_kernel(const uint8_t *__restrict__ src, int sstride, int w, int h,
		uint8_t *__restrict__ dst, int dstride, int w2, int h2, int ws, int hs,
		int src_row0, int dst_row_first, int dst_rows, int h1_total) {
	/* rows are expressed in destination-plane coordinates (-1 .. h2) of the whole component;
	 * this launch renders rows [dst_row_first, dst_row_first + dst_rows) from a source slab
	 * whose first pixel row is src_row0 (multi-GPU slabs); single GPU: src_row0 = 0. */
	int x = blockIdx.x * blockDim.x + threadIdx.x - 1;
	int yy = blockIdx.y * blockDim.y + threadIdx.y;
	if (x > w2 || yy >= dst_rows) return;
	int y = dst_row_first + yy;
	int w1 = (w + ws - 1) / ws;
	int cx = min(max(x, 0), w1 - 1), cy = min(max(y, 0), h1_total - 1);
	int hh2 = min(hs, h - cy * hs), ww2 = min(ws, w - cx * ws);
	const uint8_t *p = src + (size_t)(cy * hs - src_row0 + 1) * sstride + QS_PLANE_PAD + cx * ws;
	int sum = 0;
	for (int j = 0; j < hh2; j++) for (int i = 0; i < ww2; i++) sum += p[(size_t)j * sstride + i];
	int div = ww2 * hh2;
	dst[(size_t)(yy) * dstride + QS_PLANE_PAD + x] = (uint8_t)((sum + div / 2) / div);
	(void)h2;
}

/* ------------------------------------------------------------------------------------------
 * upsample_row, quantsmooth.h:2134-2158 (scale) + 2364-2389 (emit); one thread per chroma
 * pixel, writes ws x hs output pixels.  Edge replication of 2390-2393 / 2729-2730 is done
 * by clamping coordinates: one thread per OUTPUT-plane "cell" (x < wcells, y < hcells)
 * where cells beyond (w1, h1) replicate the last column / row.
 * ------------------------------------------------------------------------------------------ */
__global__ void qs_upsample_kernel(const uint8_t *__restrict__ C, const uint8_t *__restrict__ Yd, int cstride,
		const uint8_t *__restrict__ Yf, int ystride, uint8_t *__restrict__ out, int ostride,
		int w1, int h1, int ws, int hs, int ww, int hh, int oy0) {
	/* oy0 = first output (luma) pixel row of this slab inside the whole component: planes and
	 * `out` are slab-local, w1/h1 are whole-image quantities (0 for a single-GPU run).
	 * One thread per CELL of ws x hs output pixels: the 3x3 regression of its chroma pixel
	 * (scale, offset) is computed once and applied to the cell's luma pixels, like the reference's
	 * loop nest; cells beyond (w1, h1) replicate the last column / row (all their pixels read the
	 * last valid luma column / row and the last chroma pixel, exactly what clamping every output
	 * coordinate gives). */
	int cx = blockIdx.x * blockDim.x + threadIdx.x;     /* cell */
	int cy = blockIdx.y * blockDim.y + threadIdx.y;
	if (cx * ws >= ww || cy * hs >= hh) return;
	int sx0 = min(cx * ws, w1 * ws - 1);
	int x = sx0 / ws;                                   /* chroma pixel of this cell */
	int sy0 = min(cy * hs + oy0, h1 * hs - 1) - oy0;
	int y = (sy0 + oy0) / hs - oy0 / hs;
	const uint8_t *pc = C + (size_t)(y + 1) * cstride + QS_PLANE_PAD + x;
	const uint8_t *pd = Yd + (size_t)(y + 1) * cstride + QS_PLANE_PAD + x;
	int sA, sB;
	float scale = qs_regress(pd, pc, cstride, sA, sB);
	float offset = FA(FS((float)pc[0], FM((float)pd[0], scale)), 0.5f);
	for (int j = 0; j < hs; j++) {
		int oy = cy * hs + j;
		if (oy >= hh) break;
		int sy = min(oy + oy0, h1 * hs - 1) - oy0;
		for (int i = 0; i < ws; i++) {
			int ox = cx * ws + i;
			if (ox >= ww) break;
			int sx = min(ox, w1 * ws - 1);
			float yv = (float)Yf[(size_t)(sy + 1) * ystride + QS_PLANE_PAD + sx];
			int a = qs_cvtt_x86(FA(FM(yv, scale), offset));
			out[(size_t)oy * ostride + ox] = (uint8_t)min(max(a, 0), 255);
		}
	}
}

/* FDCT of the up-sampled plane into new coefficient arrays, quantsmooth.h:2735-2750 */
__global__ void qs_fdct_plane_kernel(const uint8_t *__restrict__ px, int pstride, int16_t *__restrict__ coef,
		int W, int nblocks) {
	int b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= nblocks) return;
	int by = b / W, bx = b - by * W;
	const uint8_t *p = px + (size_t)by * 8 * pstride + bx * 8;
	float f[64];
#pragma unroll
	for (int y = 0; y < 8; y++) {
		uint2 w = *(const uint2 *)(p + (size_t)y * pstride);
#pragma unroll
		for (int x = 0; x < 4; x++) {
			f[y * 8 + x] = (float)((int)((w.x >> (8 * x)) & 0xff) - 128);
			f[y * 8 + 4 + x] = (float)((int)((w.y >> (8 * x)) & 0xff) - 128);
		}
	}
	qs_fdct_8x8(f);
	int4 *o = (int4 *)(coef + (size_t)b * 64);
#pragma unroll
	for (int j = 0; j < 8; j++) {
		int c[8];
#pragma unroll
		for (int k = 0; k < 8; k++) c[k] = (short)qs_cvtt_x86(roundf(f[j * 8 + k]));
		o[j] = make_int4((c[0] & 0xffff) | (c[1] << 16), (c[2] & 0xffff) | (c[3] << 16),
				(c[4] & 0xffff) | (c[5] << 16), (c[6] & 0xffff) | (c[7] << 16));
	}
}

/* ------------------------------------------------------------------------------------------
 * Sharded runs (one image cut into MCU-row slabs over several GPUs, qs_cuda.cu run_slab).
 *
 * qs_stop_fixup_kernel: the component whose coefficients overflowed is "clamped only"
 * (quantsmooth.h:2602-2610 + 2670-2689): decided on the device from the run's flags.
 *
 * qs_xchg_push_kernel / qs_xchg_pull_kernel: the one neighbour exchange of the path
 * (SURVEY.md 8e).  After an IDCT pass every rank stores its first / last pixel row of every
 * plane straight into the neighbours' mailboxes - peer memory over NVLink (P2P mapping inside a
 * process, CUDA IPC between processes) - then publishes a sequence number there; the pull
 * kernel waits for its own mailbox's sequence numbers and moves the rows into the halo rows of
 * the planes.  No host thread, no stream event and no NCCL call sits between the IDCT pass and
 * the smoothing pass; mailboxes are double buffered by sequence parity, which is all the
 * write-after-read protection the stream order of the neighbours leaves to do.  The first
 * exchange of a phase also carries the "coefficient out of range" masks to every rank (OR).
 * ------------------------------------------------------------------------------------------ */
__global__ void qs_stop_fixup_kernel(const QsJob *__restrict__ jobs, int njobs, const int *__restrict__ bad) {
	for (int j = 0; j < njobs; j++) {
		const QsJob *job = jobs + j;
		if (qs_job_state(job, bad) != 1) continue;
		size_t n = (size_t)job->nblocks * 32;               /* coefficient pairs */
		uint32_t *p = (uint32_t *)job->coef;
		for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
			uint32_t w = p[i];
			int a = (short)(w & 0xffff), c = (int)w >> 16;
			a = min(max(a, -1023), 1023); c = min(max(c, -1023), 1023);
			p[i] = (uint32_t)(a & 0xffff) | ((uint32_t)c << 16);
		}
	}
}

__device__ __forceinline__ void qs_copy_row(const uint8_t *src, uint8_t *dst, uint32_t bytes) {
	/* plane rows start 8-byte aligned and are a multiple of 8 bytes long (QS_PLANE_STRIDE) */
	const uint2 *s = (const uint2 *)src; uint2 *d = (uint2 *)dst;
	for (uint32_t i = threadIdx.x; i < bytes / 8; i += blockDim.x) d[i] = s[i];
}

__global__ void __launch_bounds__(512) qs_xchg_push_kernel(const __grid_constant__ QsXchgPush a) {
	for (int r = 0; r < a.nrows; r++) qs_copy_row(a.rows[r].src, a.rows[r].dst, a.rows[r].bytes);
	for (int i = threadIdx.x; i < a.bad_n * a.npeers; i += blockDim.x)
		a.bad_dst[i / a.bad_n][i % a.bad_n] = (uint32_t)a.bad_src[i % a.bad_n];
	__threadfence_system();                                  /* every thread: its own peer stores first */
	__syncthreads();
	if (threadIdx.x < 2 && a.flag[threadIdx.x]) *(volatile uint32_t *)a.flag[threadIdx.x] = a.seq;
	if (threadIdx.x >= 32 && threadIdx.x < 32 + a.npeers && a.bad_n)
		*(volatile uint32_t *)a.bad_flag[threadIdx.x - 32] = a.seq;
	__threadfence_system();
}

__device__ __forceinline__ bool qs_wait_seq(const uint32_t *flag, uint32_t seq) {
	unsigned long long t0 = 0, t; int spins = 0;
	for (;;) {
		uint32_t v;
		asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
		if ((int32_t)(v - seq) >= 0) return true;
		if (++spins < 64) continue;
		spins = 0;
		asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
		if (!t0) t0 = t;
		if (t - t0 > 10000000000ull) return false;          /* 10 s: the peer is gone */
		__nanosleep(200);
	}
}

__global__ void __launch_bounds__(512) qs_xchg_pull_kernel(const __grid_constant__ QsXchgPull a) {
	__shared__ int ok;
	if (threadIdx.x == 0) ok = 1;
	__syncthreads();
	/* on a timeout the mapped host words say which wait it was: [0] = 1, [1] = 1 + waiter (0/1 = halo
	 * flag from the upper / lower neighbour, 32 + p = mask message of the p-th peer), [2] = the
	 * sequence number expected, [3] = the one found */
	if (threadIdx.x < 2 && a.flag[threadIdx.x] && !qs_wait_seq(a.flag[threadIdx.x], a.seq)) {
		ok = 0;
		if (a.timeout_flag) { a.timeout_flag[1] = 1 + threadIdx.x; a.timeout_flag[2] = (int)a.seq; a.timeout_flag[3] = (int)*(const volatile uint32_t *)a.flag[threadIdx.x]; }
	}
	if (threadIdx.x >= 32 && threadIdx.x < 32 + a.npeers && a.bad_n && !qs_wait_seq(a.bad_flag[threadIdx.x - 32], a.seq)) {
		ok = 0;
		if (a.timeout_flag) { a.timeout_flag[1] = 1 + threadIdx.x; a.timeout_flag[2] = (int)a.seq; a.timeout_flag[3] = (int)*(const volatile uint32_t *)a.bad_flag[threadIdx.x - 32]; }
	}
	__syncthreads();
	if (!ok) { if (threadIdx.x == 0 && a.timeout_flag) { *(volatile int *)a.timeout_flag = 1; __threadfence_system(); } return; }
	for (int r = 0; r < a.nrows; r++) qs_copy_row(a.rows[r].src, a.rows[r].dst, a.rows[r].bytes);
	for (int i = threadIdx.x; i < a.bad_n; i += blockDim.x) {
		int v = a.bad_io[i];
		for (int p = 0; p < a.npeers; p++) v |= (int)*(const volatile uint32_t *)&a.bad_in[p][i];
		a.bad_io[i] = v;
	}
}

/* grid-stride kernels are sized to the device: a few CTAs per SM */
static int qs_num_sms(void) {
	int dev = 0, n = 0;
	if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
		n = 132;
	return n;
}

cudaError_t qs_launch_stop_fixup(const QsJob *jobs_dev, int njobs, const int *bad, cudaStream_t st) {
	if (njobs <= 0) return cudaSuccess;
	qs_stop_fixup_kernel<<<qs_num_sms() * 4, 256, 0, st>>>(jobs_dev, njobs, bad);
	return cudaGetLastError();
}
cudaError_t qs_launch_xchg(const QsXchgPush *push, const QsXchgPull *pull, cudaStream_t st) {
	qs_xchg_push_kernel<<<1, 512, 0, st>>>(*push);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return e;
	qs_xchg_pull_kernel<<<1, 512, 0, st>>>(*pull);
	return cudaGetLastError();
}

/* ------------------------------------------------------------------------------------------
 * Control-data movers.  Job lists and the "coefficient out of range" flags are a few hundred
 * bytes, but as cudaMemcpyAsync they queue on the copy engines BEHIND the bulk coefficient
 * transfers of the host entry points (a 4-byte flag read would wait for a whole bulk
 * download).  Kernel parameters and stores to mapped pinned memory do not touch the copy engines.
 * ------------------------------------------------------------------------------------------ */
struct QsJobPack { QsJob j[QS_JOB_PACK]; };
__global__ void qs_store_jobs_kernel(const __grid_constant__ QsJobPack pack, QsJob *__restrict__ dst, int n) {
	int i = threadIdx.x;
	if (i < n) dst[i] = pack.j[i];
}
__global__ void qs_copy_flags_kernel(const int *__restrict__ src, volatile int *dst, int n) {
	for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
	__threadfence_system();
}
/* quant constants of the stream-ordered entry point: ~1.5 KB per record, as many per launch as
 * the 32 KB parameter space of sm_90 holds */
struct QsQuantPack { QsQuantDev q[QS_QUANT_PACK]; };
static_assert(sizeof(QsQuantPack) + sizeof(void *) + sizeof(int) <= 32764, "QS_QUANT_PACK exceeds the kernel parameter space");
static_assert(sizeof(QsQuantDev) % 4 == 0, "QsQuantDev is copied as 32-bit words");
__global__ void __launch_bounds__(256) qs_store_quant_kernel(const __grid_constant__ QsQuantPack pack,
		QsQuantDev *__restrict__ dst, int n) {
	const uint32_t *s = (const uint32_t *)pack.q;
	uint32_t *d = (uint32_t *)dst;
	for (int i = threadIdx.x; i < n * (int)(sizeof(QsQuantDev) / 4); i += blockDim.x) d[i] = s[i];
}
/* end of a stream-ordered run: per image, stop = the host's stop | the out-of-range flags of its
 * iterating components, upsampled = the full-resolution luma plane was kept and nothing stopped */
__global__ void qs_async_status_kernel(const __grid_constant__ QsStatusPack p, int n, const int *__restrict__ flags,
		int2 *__restrict__ status) {
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const QsStatusImg &m = p.img[i];
	int stop = m.host_stop;
	for (int ci = 0; ci < 16; ci++) if ((m.iter_mask >> ci) & 1) stop |= flags[m.flag0 + ci] ? 1 : 0;
	status[i] = make_int2(stop, m.kept && !stop ? 1 : 0);
}

/* ------------------------------------------------------------------------------------------
 * launch wrappers
 * ------------------------------------------------------------------------------------------ */
cudaError_t qs_set_chunks(const QsChunk *chunks, int n) {
	cudaError_t e = cudaMemcpyToSymbol(d_chunks, chunks, sizeof(QsChunk) * n);
	if (e != cudaSuccess) return e;
	return cudaMemcpyToSymbol(d_nchunks, &n, sizeof(int));
}

typedef void (*qs_smooth_fn)(const QsJob *, int, int, const float *, int *, int, int, const int *);
#define QS_V(d, lvl, wps, gs) qs_smooth_kernel<d, QS_SYNC(lvl, wps, gs)>
#ifdef QS_EXPERIMENTS
static qs_smooth_fn qs_smooth_variant(int diag, int sync, int wps) {
	if (wps == 6) {
		if (diag) return sync == 2 ? QS_V(true, 2, 6, 1) : QS_V(true, 1, 6, 1);
		return sync == 2 ? QS_V(false, 2, 6, 1) : QS_V(false, 1, 6, 1);
	}
	if (diag) return sync == 2 ? QS_V(true, 2, 4, 1) : sync ? QS_V(true, 1, 4, 1) : QS_V(true, 0, 4, 1);
	return sync == 2 ? QS_V(false, 2, 4, 1) : sync ? QS_V(false, 1, 4, 1) : QS_V(false, 0, 4, 1);
}
#else
/* the shipped configuration: lock step with one barrier per chunk, 4 warps per sub-partition
 * (the other variants were measured slower; they live behind -DQS_EXPERIMENTS) */
static qs_smooth_fn qs_smooth_variant(int diag, int, int) {
	return diag ? QS_V(true, 2, 4, 1) : QS_V(false, 2, 4, 1);
}
#endif

size_t qs_smooth_smem_bytes(int diag, int wpg) {
	return (size_t)64 * (diag ? QS_TAB_DIAG : QS_TAB_PLAIN) * 4 + (size_t)(wpg * 4) * QS_WARP_WORDS * 4;
}

cudaError_t qs_smooth_configure(void) {
#ifdef QS_EXPERIMENTS
	for (int d = 0; d < 2; d++) for (int wps = 4; wps <= 6; wps += 2)
		for (int sy = 0; sy < 3; sy++) {
			if (qs_smooth_smem_bytes(d, wps) > 227 * 1024) continue;
			cudaError_t e = cudaFuncSetAttribute(qs_smooth_variant(d, sy, wps),
					cudaFuncAttributeMaxDynamicSharedMemorySize, (int)qs_smooth_smem_bytes(d, wps));
			if (e != cudaSuccess) return e;
		}
#else
	for (int d = 0; d < 2; d++) {
		cudaError_t e = cudaFuncSetAttribute(qs_smooth_variant(d, 2, 4),
				cudaFuncAttributeMaxDynamicSharedMemorySize, (int)qs_smooth_smem_bytes(d, 4));
		if (e != cudaSuccess) return e;
	}
#endif
	return cudaSuccess;
}


cudaError_t qs_launch_idct_pass(const QsJob *jobs_dev, int njobs, int total_tiles, int mode,
		int *bad_flags, cudaStream_t st) {
	if (total_tiles <= 0) return cudaSuccess;
	int wpb = QS_IDCT_THREADS / 32;
	qs_idct_pass_kernel<<<(total_tiles + wpb - 1) / wpb, QS_IDCT_THREADS, 0, st>>>(jobs_dev, njobs, total_tiles, mode, bad_flags);
	return cudaGetLastError();
}

cudaError_t qs_launch_smooth(const QsJob *jobs_dev, int njobs, int total_tiles, const float *tables_dev,
		int *tile_counter, int flags, int clamp_out, int num_sms, int sync, int wpg, const int *bad, cudaStream_t st) {
	if (total_tiles <= 0) return cudaSuccess;
	cudaError_t e = cudaMemsetAsync(tile_counter, 0, sizeof(int), st);
	if (e != cudaSuccess) return e;
	int diag = (flags & QS_DIAGONALS) ? 1 : 0;
#ifdef QS_EXPERIMENTS
	if ((wpg != 4 && wpg != 6) || qs_smooth_smem_bytes(diag, wpg) > 227 * 1024) wpg = 4;
	if (sync < 0 || sync > 2) sync = 2;
#else
	wpg = 4; sync = 2;
#endif
	int warps = wpg * 4;
	int grid = (total_tiles + warps - 1) / warps;
	if (grid > num_sms) grid = num_sms;
	qs_smooth_variant(diag, sync, wpg)<<<grid, wpg * 128, qs_smooth_smem_bytes(diag, wpg), st>>>(
			jobs_dev, njobs, total_tiles, tables_dev, tile_counter, flags, clamp_out, bad);
	return cudaGetLastError();
}

cudaError_t qs_launch_lowq(const QsJob *jobs_dev, int njobs, int total_tiles, int flags, int clamp_out,
		const int *bad, cudaStream_t st) {
	if (total_tiles <= 0) return cudaSuccess;
	qs_lowq_kernel<<<(total_tiles + 3) / 4, 128, 0, st>>>(jobs_dev, njobs, total_tiles, flags, clamp_out, bad);
	return cudaGetLastError();
}

cudaError_t qs_launch_scale_clamp(int16_t *coef, size_t n, const QsQuantDev *qd, int dequant, int clamp,
		cudaStream_t st) {
	if (!n) return cudaSuccess;
	size_t blocks = (n + 255) / 256;
	size_t cap = (size_t)qs_num_sms() * 16;
	if (blocks > cap) blocks = cap;
	qs_scale_clamp_kernel<<<(unsigned)blocks, 256, 0, st>>>(coef, n, qd, dequant, clamp);
	return cudaGetLastError();
}

cudaError_t qs_launch_downsample(const uint8_t *src, int sstride, int w, int h, uint8_t *dst, int dstride,
		int w2, int h2, int ws, int hs, int src_row0, int dst_row_first, int dst_rows, int h1_total,
		cudaStream_t st) {
	dim3 blk(64, 4), grd((w2 + 2 + 63) / 64, (dst_rows + 3) / 4);
	/* dst points at the plane row that holds destination row dst_row_first */
	qs_downsample_kernel<<<grd, blk, 0, st>>>(src, sstride, w, h, dst, dstride, w2, h2, ws, hs,
			src_row0, dst_row_first, dst_rows, h1_total);
	return cudaGetLastError();
}

cudaError_t qs_launch_upsample(const uint8_t *C, const uint8_t *Yd, int cstride, const uint8_t *Yf, int ystride,
		uint8_t *out, int ostride, int w1, int h1, int ws, int hs, int ww, int hh, int oy0, cudaStream_t st) {
	int wc = (ww + ws - 1) / ws, hc = (hh + hs - 1) / hs;          /* cells of ws x hs output pixels */
	dim3 blk(64, 4), grd((wc + 63) / 64, (hc + 3) / 4);
	qs_upsample_kernel<<<grd, blk, 0, st>>>(C, Yd, cstride, Yf, ystride, out, ostride, w1, h1, ws, hs, ww, hh, oy0);
	return cudaGetLastError();
}

cudaError_t qs_launch_fdct_plane(const uint8_t *px, int pstride, int16_t *coef, int W, int H, cudaStream_t st) {
	int n = W * H;
	if (!n) return cudaSuccess;
	qs_fdct_plane_kernel<<<(n + 127) / 128, 128, 0, st>>>(px, pstride, coef, W, n);
	return cudaGetLastError();
}

/* ------------------------------------------------------------------------------------------
 * Render to interleaved RGB (SURVEY.md 8f row f2): what libjpeg does after the reference's
 * jpegqs_start_decompress hands the smoothed coefficients back (quantsmooth.h:2861-2904):
 * islow IDCT (already in the planes), "fancy" triangle up-sampling of sub-sampled chroma
 * (libjpeg jdsample.c h2v1_fancy_upsample / h2v2_fancy_upsample), YCbCr -> RGB with the
 * fixed-point tables of jdcolor.c.  All integer, restated from the published algorithms;
 * parity is checked against Pillow's libjpeg-turbo decode of the same file.
 * One thread per output pixel.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
	const uint8_t *plane[3];
	int stride[3];
	int cw[3], ch[3];        /* real (not block padded) component size: libjpeg downsampled_width/height */
	int hs[3], vs[3];        /* expansion factors max_samp / samp of each component */
	int ncomp, width, height, ycc;
} QsRenderArgs;

/* sample (x, y) of a padded sample plane */
struct QsPlanePx {
	const uint8_t *p; int stride;
	__device__ __forceinline__ int operator()(int x, int y) const { return p[(size_t)(y + 1) * stride + QS_PLANE_PAD + x]; }
};

/* One up-sampled sample at output pixel (ox, oy) of a component whose expansion factors are
 * hs x vs and whose real (not block padded) size is cw x ch; px(x, y) reads its sample (x, y).
 * Edges replicate the last real sample, column cw - 1 / row ch - 1, as libjpeg does.  FANCY false:
 * replication only - libjpeg's jinit_upsampler turns fancy up-sampling off when the smallest DCT
 * scaled size is 1 (scale 1/8), because its main controller has no context rows then. */
template <bool FANCY = true, class Px>
__host__ __device__ __forceinline__ int qs_upsample_at(const Px &px, int hs, int vs, int cw, int ch, int ox, int oy) {
	if (hs == 1 && vs == 1) return px(ox, oy);
	if (!FANCY) return px(min(ox / hs, cw - 1), min(oy / vs, ch - 1));
	if (hs == 2 && vs == 1 && cw > 2) {                 /* h2v1_fancy_upsample */
		int x = ox >> 1, v = px(x, oy);
		if (ox & 1) return x == cw - 1 ? v : (v * 3 + px(x + 1, oy) + 2) >> 2;
		return x == 0 ? v : (v * 3 + px(x - 1, oy) + 1) >> 2;
	}
	if (hs == 2 && vs == 2 && cw > 2) {                 /* h2v2_fancy_upsample */
		int x = ox >> 1, y = oy >> 1;
		int y1 = (oy & 1) ? min(y + 1, ch - 1) : max(y - 1, 0);   /* nearer neighbour row, edge replicated */
		int cur = px(x, y) * 3 + px(x, y1);
		if (ox & 1) {
			if (x == cw - 1) return (cur * 4 + 7) >> 4;
			return (cur * 3 + px(x + 1, y) * 3 + px(x + 1, y1) + 7) >> 4;
		}
		if (x == 0) return (cur * 4 + 8) >> 4;
		return (cur * 3 + px(x - 1, y) * 3 + px(x - 1, y1) + 8) >> 4;
	}
	if (hs == 1 && vs == 2) {                           /* h1v2_fancy_upsample (libjpeg-turbo >= 2.0) */
		int y = oy >> 1, y1 = (oy & 1) ? min(y + 1, ch - 1) : max(y - 1, 0);
		return (px(ox, y) * 3 + px(ox, y1) + ((oy & 1) ? 2 : 1)) >> 2;
	}
	return px(min(ox / hs, cw - 1), min(oy / vs, ch - 1));   /* box replication (int_upsample) */
}

/* one output pixel, r | g << 8 | b << 16: YCbCr -> RGB with the fixed-point tables of jdcolor.c
 * (build_ycc_rgb_table / ycc_rgb_convert, SCALEBITS 16) when ycc, the three samples as they are
 * otherwise (a grey image passes its sample three times) */
__host__ __device__ __forceinline__ uint32_t qs_rgb_pixel(int y, int c1, int c2, bool ycc) {
	int r = y, g = c1, b = c2;
	if (ycc) {
		int cb = c1 - 128, cr = c2 - 128;
		r = min(max(y + ((91881 * cr + 32768) >> 16), 0), 255);
		g = min(max(y + ((-22554 * cb + 32768 - 46802 * cr) >> 16), 0), 255);
		b = min(max(y + ((116130 * cb + 32768) >> 16), 0), 255);
	}
	return (uint32_t)r | ((uint32_t)g << 8) | ((uint32_t)b << 16);
}

/* Pillow's rgb2l (Convert.c, L24 >> 16) of r | g << 8 | b << 16 */
__host__ __device__ __forceinline__ uint32_t qs_luma(uint32_t v) {
	return ((v & 255) * 19595 + ((v >> 8) & 255) * 38470 + ((v >> 16) & 255) * 7471 + 0x8000) >> 16;
}

/* Pillow's MULDIV255(a, b) */
__host__ __device__ __forceinline__ int qs_muldiv255(int a, int b) {
	const int t = a * b + 128;
	return ((t >> 8) + t) >> 8;
}

/* One 4-component pixel, r | g << 8 | b << 16, as Pillow's convert("RGB") gives it.  Pillow decodes these
 * files with libjpeg's JCS_CMYK output and raw mode CMYK;I, which inverts all four samples.  YCCK: libjpeg's
 * ycck_cmyk_convert first gives 255 - (R, G, B) of the YCbCr triple and passes K through, so Pillow's C, M, Y
 * are R, G, B.  Then cmyk2rgb with nk = 255 - Pillow's K = s3: out = nk - MULDIV255(C, nk), never below 0. */
__host__ __device__ __forceinline__ uint32_t qs_cmyk_pixel(int s0, int s1, int s2, int s3, bool ycck) {
	const uint32_t cmy = ycck ? qs_rgb_pixel(s0, s1, s2, true) : 0xffffffu ^ ((uint32_t)s0 | (uint32_t)s1 << 8 | (uint32_t)s2 << 16);
	const int nk = s3;
	return (uint32_t)(nk - qs_muldiv255(cmy & 255, nk)) | (uint32_t)(nk - qs_muldiv255((cmy >> 8) & 255, nk)) << 8 |
			(uint32_t)(nk - qs_muldiv255(cmy >> 16, nk)) << 16;
}

/* the render's pixel from its up-sampled samples (s3: 4-component conversions only) by conversion CONV
 * (qs_kernels.h QS_CONV_*) */
template <int CONV>
__host__ __device__ __forceinline__ uint32_t qs_convert_pixel(int s0, int s1, int s2, int s3, bool ycc) {
	if constexpr (CONV == QS_CONV_NONE) return qs_rgb_pixel(s0, s1, s2, ycc);
	else if constexpr (CONV == QS_CONV_L) return qs_luma(qs_rgb_pixel(s0, s1, s2, ycc));
	else if constexpr (CONV == QS_CONV_CMYK_RGB) return qs_cmyk_pixel(s0, s1, s2, s3, ycc);
	else return qs_luma(qs_cmyk_pixel(s0, s1, s2, s3, ycc));
}

__global__ void qs_render_rgb_kernel(QsRenderArgs a, uint8_t *__restrict__ rgb) {
	int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y * blockDim.y + threadIdx.y;
	if (ox >= a.width || oy >= a.height) return;
	uint8_t *o = rgb + ((size_t)oy * a.width + ox) * 3;
	int y = qs_upsample_at(QsPlanePx{a.plane[0], a.stride[0]}, a.hs[0], a.vs[0], a.cw[0], a.ch[0], ox, oy), c1 = y, c2 = y;
	if (a.ncomp >= 3) {
		c1 = qs_upsample_at(QsPlanePx{a.plane[1], a.stride[1]}, a.hs[1], a.vs[1], a.cw[1], a.ch[1], ox, oy);
		c2 = qs_upsample_at(QsPlanePx{a.plane[2], a.stride[2]}, a.hs[2], a.vs[2], a.cw[2], a.ch[2], ox, oy);
	}
	uint32_t px = qs_rgb_pixel(y, c1, c2, a.ncomp >= 3 && a.ycc);
	o[0] = (uint8_t)px; o[1] = (uint8_t)(px >> 8); o[2] = (uint8_t)(px >> 16);
}

/* ------------------------------------------------------------------------------------------
 * Scaled decode (DESIGN.md section 3.9): libjpeg's reduced-size IDCTs, jidctred.c jpeg_idct_4x4,
 * jpeg_idct_2x2 and jpeg_idct_1x1, restated from the published algorithm.  They are the LL&M
 * butterfly of the islow IDCT with the terms the smaller output does not need left out, in
 * fixed point with CONST_BITS 13 and PASS1_BITS 2: jpeg_idct_4x4 reads no row or column 4,
 * jpeg_idct_2x2 only rows / columns 0, 1, 3, 5 and 7, jpeg_idct_1x1 only the DC term.
 * The descale of every output is DESCALE(x, n) = (x + 2^(n-1)) >> n.  libjpeg-turbo runs SSE2
 * versions of the 4x4 and 2x2 ones; they saturate where the C range-limit table wraps (a sample
 * beyond [-384, 383] before the +128), so these clamp, as the islow render does (section 6 f2).
 * jpeg_idct_1x1 has no SIMD version: it keeps the table's wrap.
 * ------------------------------------------------------------------------------------------ */
__host__ __device__ __forceinline__ int qs_descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

/* one 1-D pass of jpeg_idct_4x4 over in[0..7] (in[4] is not read): out[0..3] before the descale */
__host__ __device__ __forceinline__ void qs_red4_1d(const int *in, int *out) {
	const int t0 = in[0] * (1 << 14);                       /* << (CONST_BITS + 1) */
	const int t2 = in[2] * 15137 - in[6] * 6270;            /* FIX(1.847759065), FIX(0.765366865) */
	const int t10 = t0 + t2, t12 = t0 - t2;
	const int z1 = in[7], z2 = in[5], z3 = in[3], z4 = in[1];
	/* FIX(0.211164243), FIX(1.451774981), FIX(2.172734803), FIX(1.061594337) */
	const int o0 = -z1 * 1730 + z2 * 11893 - z3 * 17799 + z4 * 8697;
	/* FIX(0.509795579), FIX(0.601344887), FIX(0.899976223), FIX(2.562915447) */
	const int o2 = -z1 * 4176 - z2 * 4926 + z3 * 7373 + z4 * 20995;
	out[0] = t10 + o2; out[3] = t10 - o2; out[1] = t12 + o0; out[2] = t12 - o0;
}

/* one 1-D pass of jpeg_idct_2x2 over in[0, 1, 3, 5, 7]: out[0..1] before the descale */
__host__ __device__ __forceinline__ void qs_red2_1d(const int *in, int *out) {
	const int t10 = in[0] * (1 << 15);                      /* << (CONST_BITS + 2) */
	/* FIX(0.720959822), FIX(0.850430095), FIX(1.272758580), FIX(3.624509785) */
	const int t0 = -in[7] * 5906 + in[5] * 6967 - in[3] * 10426 + in[1] * 29692;
	out[0] = t10 + t0; out[1] = t10 - t0;
}

/* libjpeg's post-IDCT range limit (prepare_range_limit_table): the low 10 bits of x as a signed value,
 * plus 128, clamped to [0, 255] */
__host__ __device__ __forceinline__ int qs_range_limit(int x) {
	x &= 1023;
	return x < 128 ? x + 128 : x < 512 ? 255 : x < 896 ? 0 : x - 896;
}

__host__ __device__ __forceinline__ void qs_store_u32(uint8_t *d, uint32_t v) {
#ifdef __CUDA_ARCH__
	*(uint32_t *)d = v;
#else
	memcpy(d, &v, 4);
#endif
}

/* the ss x ss samples of one block at DCT scaled size ss into dst (row stride `stride`).  cf: the 64
 * de-quantized coefficients in natural order (only cf[0] is read for ss 1).  ss 8 is the islow IDCT of
 * the full-size render. */
__host__ __device__ __forceinline__ void qs_idct_scaled(const int *cf, int ss, uint8_t *dst, int stride) {
	if (ss == 8) {
		int ws[64];
#pragma unroll
		for (int x = 0; x < 8; x++) {
			int in[8], o[8];
#pragma unroll
			for (int y = 0; y < 8; y++) in[y] = cf[y * 8 + x];
			qs_islow_1d<1024>(in, o);
#pragma unroll
			for (int y = 0; y < 8; y++) ws[y * 8 + x] = o[y] >> 11;
		}
		uint32_t rlo[8], rhi[8];
		qs_islow_rows(ws, rlo, rhi);
#pragma unroll
		for (int y = 0; y < 8; y++) { qs_store_u32(dst + y * stride, rlo[y]); qs_store_u32(dst + y * stride + 4, rhi[y]); }
	} else if (ss == 4) {
		int ws[32];                                         /* [4 rows][8 columns]; column 4 unused */
#pragma unroll
		for (int x = 0; x < 8; x++) {
			if (x == 4) { for (int y = 0; y < 4; y++) ws[y * 8 + x] = 0; continue; }
			int in[8], o[4];
#pragma unroll
			for (int y = 0; y < 8; y++) in[y] = cf[y * 8 + x];
			qs_red4_1d(in, o);
#pragma unroll
			for (int y = 0; y < 4; y++) ws[y * 8 + x] = qs_descale(o[y], 12);   /* CONST_BITS - PASS1_BITS + 1 */
		}
#pragma unroll
		for (int y = 0; y < 4; y++) {
			int o[4];
			qs_red4_1d(ws + y * 8, o);
			qs_store_u32(dst + y * stride, qs_pack_sat_u8(qs_descale(o[0], 19) + 128, qs_descale(o[1], 19) + 128,
					qs_descale(o[2], 19) + 128, qs_descale(o[3], 19) + 128));        /* CONST_BITS + PASS1_BITS + 3 + 1 */
		}
	} else if (ss == 2) {
		int ws[16];                                         /* [2 rows][8 columns]; columns 2, 4, 6 unused */
#pragma unroll
		for (int x = 0; x < 8; x++) {
			if (x == 2 || x == 4 || x == 6) { ws[x] = ws[8 + x] = 0; continue; }
			int in[8], o[2];
#pragma unroll
			for (int y = 0; y < 8; y++) in[y] = cf[y * 8 + x];
			qs_red2_1d(in, o);
			ws[x] = qs_descale(o[0], 13); ws[8 + x] = qs_descale(o[1], 13);       /* CONST_BITS - PASS1_BITS + 2 */
		}
#pragma unroll
		for (int y = 0; y < 2; y++) {
			int o[2];
			qs_red2_1d(ws + y * 8, o);
			const int a = qs_descale(o[0], 20) + 128, b = qs_descale(o[1], 20) + 128;   /* CONST_BITS + PASS1_BITS + 3 + 2 */
			dst[y * stride] = (uint8_t)(a < 0 ? 0 : a > 255 ? 255 : a);
			dst[y * stride + 1] = (uint8_t)(b < 0 ? 0 : b > 255 ? 255 : b);
		}
	} else {
		dst[0] = (uint8_t)qs_range_limit(qs_descale(cf[0], 3));
	}
}

/* ------------------------------------------------------------------------------------------
 * Stream-ordered render (qs_cuda.cu jpegqs_cuda_render_async): coefficients -> islow IDCT ->
 * libjpeg's up-sampling -> colour conversion -> pixels in one launch per batch; no sample plane
 * goes through global memory.  A CTA renders one QS_RENDER_TW x QS_RENDER_TH tile of output
 * pixels.  It IDCTs into shared memory every block of every component under the tile, plus the
 * blocks holding the one-sample ring the fancy up-sampler reads, then computes the tile's pixels
 * from there.  Per component the window is at most 16 x 8 blocks: 16 x 8 at full resolution, 10 x 6
 * with 2:1 sub-sampling and its ring, fewer for 3:1 and 4:1 (which replicate and need no ring).
 * Coefficients are only read; de-quantization happens in registers, in int32 (jidctint.c).
 * Scaled decode (D = scale_denom 2, 4 or 8): the tile is still 128 x 64 output pixels and the windows
 * hold samples at each component's DCT scaled size (QsRenderImg.lss), so a tile reads up to D^2 times
 * the blocks; each block gives ss x ss samples through qs_idct_scaled.  D = 1 is the code above,
 * unchanged.
 * ------------------------------------------------------------------------------------------ */
#define QS_RT_THREADS 256
#define QS_RS_W 128
#define QS_RS_H 64
static_assert(QS_RENDER_TW == 128 && QS_RENDER_TH == 64, "the shared sample window is sized for 128 x 64 tiles");

struct QsRenderPack { QsRenderImg img[QS_RENDER_PACK]; };
static_assert(sizeof(QsRenderImg) == 496, "orient sits in the padding before q");
static_assert(sizeof(QsRenderPack) + 2 * sizeof(void *) + 2 * sizeof(int) <= 32764,
		"QS_RENDER_PACK exceeds the kernel parameter space");
struct QsRenderPack4 { QsRenderImg4 img[QS_RENDER_PACK4]; };
static_assert(sizeof(QsRenderImg4) == 624, "QsRenderImg4 has no padding");
static_assert(sizeof(QsRenderPack4) + 2 * sizeof(void *) + 2 * sizeof(int) <= 32764 &&
		sizeof(QsRenderPack4) + sizeof(QsRenderImg4) + 2 * sizeof(void *) + 2 * sizeof(int) > 32764,
		"QS_RENDER_PACK4 is the most 4-component descriptors the kernel parameter space holds");
/* the kernel's descriptors: 4 components for the CMYK conversions, QsRenderImg otherwise */
template <int CONV> using QsRenderPackOf = std::conditional_t<(CONV >= QS_CONV_CMYK_RGB), QsRenderPack4, QsRenderPack>;

/* sample (x, y) of a component's shared window whose first sample is (x0, y0) */
struct QsSmemPx {
	const uint8_t *s; int x0, y0;
	__device__ __forceinline__ int operator()(int x, int y) const { return s[(y - y0) * QS_RS_W + (x - x0)]; }
};

struct QsRenderComp { const int16_t *coef; int wblk, bx0, by0, nbx, nby, cw, ch, hs, vs; };

/* the oriented store's staging (orientations 5..8): one byte plane per channel of the tile's 64 rows, each
 * padded to an odd pitch so that the column reads of a half-warp fall in different banks */
#define QS_RT_TB_PITCH (QS_RENDER_TW + 1)
#define QS_RT_TB_PLANE (QS_RENDER_TH * QS_RT_TB_PITCH)
#define QS_RT_TB_BYTES (3 * QS_RT_TB_PLANE)

/* pixels px[0 .. cnt) (cnt >= 4: all four) to the consecutive output pixels pos, pos + 1, ...; plane: the
 * pixels of one CHW plane.  Aligned groups of four go out as 32-bit words. */
template <int STORE>
__device__ __forceinline__ void qs_render_store4(uint8_t *out, size_t plane, size_t pos, const uint32_t px[4], int cnt) {
	if (STORE == QS_RENDER_HWC) {
		uint8_t *o = out + pos * 3;
		if (cnt >= 4 && !((uintptr_t)o & 3)) {
			uint32_t *o4 = (uint32_t *)o;
			o4[0] = px[0] | (px[1] << 24);
			o4[1] = (px[1] >> 8) | (px[2] << 16);
			o4[2] = (px[2] >> 16) | (px[3] << 8);
		} else {
			for (int i = 0; i < 4 && i < cnt; i++) {
				o[3 * i] = (uint8_t)px[i]; o[3 * i + 1] = (uint8_t)(px[i] >> 8); o[3 * i + 2] = (uint8_t)(px[i] >> 16);
			}
		}
	} else {
#pragma unroll
		for (int k = 0; k < (STORE == QS_RENDER_GREY ? 1 : 3); k++) {
			uint8_t *o = out + (size_t)k * plane + pos;
			if (cnt >= 4 && !((uintptr_t)o & 3)) {
				*(uint32_t *)o = __byte_perm(__byte_perm(px[0], px[1], 0x0040 + 0x0011 * k),
						__byte_perm(px[2], px[3], 0x0040 + 0x0011 * k), 0x5410);
			} else {
				for (int i = 0; i < 4 && i < cnt; i++) o[i] = (uint8_t)(px[i] >> (8 * k));
			}
		}
	}
}

/* STORE: QS_RENDER_HWC / QS_RENDER_CHW (three bytes per pixel), or QS_RENDER_GREY (one byte per pixel,
 * the CHW store of plane 0 only; for 1-component images).  D: the scale denominator (1, 2, 4, 8); the
 * descriptors then hold the scaled geometry (qs_render_images).  ORIENTED: some image of the launch has an
 * orientation other than 1; without it the kernel holds only the unoriented store.  CONV: the colour
 * conversion (qs_kernels.h QS_CONV_*); the CMYK ones read QsRenderImg4 descriptors and a fourth window,
 * NONE is the file's own colour and compiles to the kernel it was before the conversions existed. */
template <int STORE, int D, bool ORIENTED, int CONV = QS_CONV_NONE>
__global__ void __launch_bounds__(QS_RT_THREADS, 2) qs_render_async_kernel(const __grid_constant__ QsRenderPackOf<CONV> p,
		int n, const int2 *__restrict__ status) {
	constexpr int NC = CONV >= QS_CONV_CMYK_RGB ? 4 : 3;  /* windows */
	__shared__ __align__(16) uint8_t pix[NC][QS_RS_H * QS_RS_W];
	__shared__ int qmul[NC][64];
	__shared__ QsRenderComp g[NC];
	__shared__ int glss[NC];                             /* D > 1: log2 of each window's DCT scaled size */
	const int tile = blockIdx.x;
	int lo = 0, hi = n - 1;
	while (lo < hi) {                                    /* last image with tile_begin <= tile */
		int mid = (lo + hi + 1) >> 1;
		if (p.img[mid].tile_begin <= tile) lo = mid; else hi = mid - 1;
	}
	const auto &im = p.img[lo];
	const int W = im.width, H = im.height, nc = im.ncomp, ntx = (W + QS_RENDER_TW - 1) / QS_RENDER_TW;
	const int t = tile - im.tile_begin, x0 = (t % ntx) * QS_RENDER_TW, y0 = (t / ntx) * QS_RENDER_TH;
	const int x1 = min(x0 + QS_RENDER_TW, W) - 1, y1 = min(y0 + QS_RENDER_TH, H) - 1;   /* last pixel of the tile */
	if (threadIdx.x < nc) {
		const int c = threadIdx.x;
		/* components 1 and 2 of an up-sampled image: coef_up, at component 0's geometry */
		bool up = false;
		if constexpr (NC == 3) up = c > 0 && (im.up_mode == 1 || (im.up_mode == 2 && status[lo].y != 0));
		const int k = up ? 0 : c;
		QsRenderComp r;
		if constexpr (NC == 3) r.coef = up ? im.coef_up[c - 1] : im.coef[c];
		else r.coef = im.coef[c];
		r.wblk = im.wblk[k]; r.cw = im.cw[k]; r.ch = im.ch[k]; r.hs = im.hs[k]; r.vs = im.vs[k];
		const int rx = r.hs == 2 ? 1 : 0, ry = r.vs == 2 ? 1 : 0;     /* the fancy up-sampler's ring */
		const int lss = D == 1 ? 3 : (im.lss >> (2 * k)) & 3;
		r.bx0 = max(x0 / r.hs - rx, 0) >> lss; r.nbx = (min(x1 / r.hs + rx, r.cw - 1) >> lss) - r.bx0 + 1;
		r.by0 = max(y0 / r.vs - ry, 0) >> lss; r.nby = (min(y1 / r.vs + ry, r.ch - 1) >> lss) - r.by0 + 1;
		g[c] = r;
		if (D > 1) glss[c] = lss;
	}
	for (int i = threadIdx.x; i < nc * 64; i += QS_RT_THREADS) qmul[i >> 6][i & 63] = im.q[i >> 6][i & 63];
	__syncthreads();

	/* islow IDCT (D > 1: each window's scaled IDCT) of every block of the windows, one thread per block
	 * (as qs_idct_pass_kernel) */
	const int nb0 = g[0].nbx * g[0].nby, nb1 = nc > 1 ? g[1].nbx * g[1].nby : 0, nb2 = nc > 2 ? g[2].nbx * g[2].nby : 0;
	const int nb3 = NC == 4 ? g[NC - 1].nbx * g[NC - 1].nby : 0;
	for (int k = threadIdx.x; k < nb0 + nb1 + nb2 + nb3; k += QS_RT_THREADS) {
		int c = k < nb0 ? 0 : k < nb0 + nb1 ? 1 : 2;
		int j = k - (c == 0 ? 0 : c == 1 ? nb0 : nb0 + nb1);
		if (NC == 4 && j >= nb2 && c == 2) { c = 3; j -= nb2; }
		const QsRenderComp &r = g[c];
		const int lby = j / r.nbx, lbx = j - lby * r.nbx;
		const int4 *src = (const int4 *)(r.coef + ((size_t)(r.by0 + lby) * r.wblk + r.bx0 + lbx) * 64);
		if constexpr (D > 1) {
			if (glss[c] == 0) {                             /* jpeg_idct_1x1: the DC term only */
				int cf0 = __ldg((const short *)src) * qmul[c][0];
				qs_idct_scaled(&cf0, 1, &pix[c][lby * QS_RS_W + lbx], QS_RS_W);
				continue;
			}
		}
		int cf[64];
#pragma unroll
		for (int v8 = 0; v8 < 8; v8++) {
			int4 v = __ldg(src + v8);
			int w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
			for (int h = 0; h < 4; h++) {
				cf[v8 * 8 + 2 * h] = (short)(w[h] & 0xffff) * qmul[c][v8 * 8 + 2 * h];
				cf[v8 * 8 + 2 * h + 1] = (w[h] >> 16) * qmul[c][v8 * 8 + 2 * h + 1];
			}
		}
		if constexpr (D > 1) {
			const int lss = glss[c];
			qs_idct_scaled(cf, 1 << lss, &pix[c][((lby * QS_RS_W) + lbx) << lss], QS_RS_W);
		} else {
			int ws[64];
#pragma unroll
			for (int x = 0; x < 8; x++) {
				int in[8], o[8];
#pragma unroll
				for (int y = 0; y < 8; y++) in[y] = cf[y * 8 + x];
				qs_islow_1d<1024>(in, o);
#pragma unroll
				for (int y = 0; y < 8; y++) ws[y * 8 + x] = o[y] >> 11;
			}
			uint32_t rlo[8], rhi[8];
			qs_islow_rows(ws, rlo, rhi);
			uint8_t *d = &pix[c][lby * 8 * QS_RS_W + lbx * 8];
#pragma unroll
			for (int y = 0; y < 8; y++) *(uint2 *)(d + y * QS_RS_W) = make_uint2(rlo[y], rhi[y]);
		}
	}
	__syncthreads();

	/* pixels: a warp renders a row of 128, four consecutive pixels per lane */
	const int ls0 = D == 1 ? 3 : glss[0], ls1 = D == 1 ? 3 : glss[1], ls2 = D == 1 ? 3 : glss[2];
	const QsSmemPx P0{pix[0], g[0].bx0 << ls0, g[0].by0 << ls0}, P1{pix[1], g[1].bx0 << ls1, g[1].by0 << ls1},
			P2{pix[2], g[2].bx0 << ls2, g[2].by0 << ls2};
	const int lane = threadIdx.x & 31;
	const bool ycc = nc >= 3 && im.ycc;
	const size_t plane = (size_t)W * H;
	auto pixel = [&](int x, int y) -> uint32_t {
		const int l = qs_upsample_at<D != 8>(P0, g[0].hs, g[0].vs, g[0].cw, g[0].ch, x, y);
		int c1 = l, c2 = l;
		if (nc >= 3) {
			c1 = qs_upsample_at<D != 8>(P1, g[1].hs, g[1].vs, g[1].cw, g[1].ch, x, y);
			c2 = qs_upsample_at<D != 8>(P2, g[2].hs, g[2].vs, g[2].cw, g[2].ch, x, y);
		}
		int c3 = 0;
		if constexpr (NC == 4) {
			const int ls3 = D == 1 ? 3 : glss[3];
			const QsSmemPx P3{pix[3], g[3].bx0 << ls3, g[3].by0 << ls3};
			c3 = qs_upsample_at<D != 8>(P3, g[3].hs, g[3].vs, g[3].cw, g[3].ch, x, y);
		}
		return qs_convert_pixel<CONV>(l, c1, c2, c3, ycc);
	};
	const int orient = ORIENTED ? im.orient : 1;         /* CTA-uniform */
	if (!ORIENTED || orient < 5) {
		/* 1 and the flips: a lane renders four consecutive pixels of an output row, output columns c0..c1
		 * holding the tile's source columns x0..x1 (mirrored for 2 and 3), from output row oy or H-1-oy */
		auto rows = [&](auto flips) {
			constexpr bool F = decltype(flips)::value;
			const bool mx = F && (orient == 2 || orient == 3), my = F && (orient == 3 || orient == 4);
			const int c0 = mx ? W - 1 - x1 : x0, c1 = mx ? W - 1 - x0 : x1, oc = c0 + lane * 4;
			if (oc > c1) return;
			for (int oy = y0 + (threadIdx.x >> 5); oy <= y1; oy += QS_RT_THREADS / 32) {
				uint32_t px[4];
#pragma unroll
				for (int i = 0; i < 4; i++) {
					const int c = min(oc + i, c1);
					px[i] = pixel(mx ? W - 1 - c : c, oy);
				}
				qs_render_store4<STORE>(im.out, plane, (size_t)(my ? H - 1 - oy : oy) * W + oc, px, c1 - oc + 1);
			}
		};
		if (orient <= 1) rows(std::false_type());       /* unoriented: the flips compile away */
		else rows(std::true_type());
		return;
	}
	if constexpr (ORIENTED) {
		/* 5..8 swap the axes: the tile's pixels go to tb (QS_RT_TB_BYTES of dynamic shared memory, one byte
		 * plane per channel, QS_RT_TB_PITCH bytes per row), then every source column x0..x1 is written as
		 * part of output row x (5, 6) or W-1-x (7, 8), a half-warp per row and four pixels per lane, so the
		 * global stores stay row-contiguous.  The output is H pixels wide. */
		extern __shared__ __align__(16) uint8_t tb[];
		constexpr int NK = STORE == QS_RENDER_GREY ? 1 : 3;
		const int ox = x0 + lane * 4;
		if (ox <= x1)
			for (int oy = y0 + (threadIdx.x >> 5); oy <= y1; oy += QS_RT_THREADS / 32) {
				uint8_t *row = tb + (oy - y0) * QS_RT_TB_PITCH + (ox - x0);
#pragma unroll
				for (int i = 0; i < 4; i++) {
					const uint32_t v = pixel(min(ox + i, x1), oy);
#pragma unroll
					for (int k = 0; k < NK; k++) row[k * QS_RT_TB_PLANE + i] = (uint8_t)(v >> (8 * k));
				}
			}
		__syncthreads();
		const bool mc = orient == 6 || orient == 7, mr = orient == 7 || orient == 8;
		const int c0 = mc ? H - 1 - y1 : y0, c1 = mc ? H - 1 - y0 : y1, oc = c0 + (threadIdx.x & 15) * 4;
		if (oc > c1) return;
		for (int r = threadIdx.x >> 4; r <= x1 - x0; r += QS_RT_THREADS / 16) {
			uint32_t px[4];
#pragma unroll
			for (int i = 0; i < 4; i++) {
				const int c = min(oc + i, c1);
				const uint8_t *s = tb + ((mc ? H - 1 - c : c) - y0) * QS_RT_TB_PITCH + r;
				px[i] = s[0];
				if (NK == 3) px[i] |= (uint32_t)s[QS_RT_TB_PLANE] << 8 | (uint32_t)s[2 * QS_RT_TB_PLANE] << 16;
			}
			const int orow = mr ? W - 1 - (x0 + r) : x0 + r;
			qs_render_store4<STORE>(im.out, plane, (size_t)orow * H + oc, px, c1 - oc + 1);
		}
	}
}

/* the store modes each conversion is instantiated for: the RGB ones HWC and CHW (NONE also GREY for grey
 * images), the luma ones GREY; the callers pass no other pair */
template <int D, bool O, int CONV>
static void qs_launch_render_store(const QsRenderPackOf<CONV> &pack, int n, int tiles, const int2 *status, int store,
		size_t smem, cudaStream_t st) {
	if constexpr (CONV == QS_CONV_NONE || CONV == QS_CONV_CMYK_RGB) {
		if (store == QS_RENDER_HWC) qs_render_async_kernel<QS_RENDER_HWC, D, O, CONV><<<tiles, QS_RT_THREADS, smem, st>>>(pack, n, status);
		else if (store == QS_RENDER_CHW) qs_render_async_kernel<QS_RENDER_CHW, D, O, CONV><<<tiles, QS_RT_THREADS, smem, st>>>(pack, n, status);
		else if constexpr (CONV == QS_CONV_NONE) qs_render_async_kernel<QS_RENDER_GREY, D, O><<<tiles, QS_RT_THREADS, smem, st>>>(pack, n, status);
	} else {
		qs_render_async_kernel<QS_RENDER_GREY, D, O, CONV><<<tiles, QS_RT_THREADS, smem, st>>>(pack, n, status);
	}
}

/* oriented: some image has an orientation other than 1; smem: the staging of 5..8, or 0 */
template <int D, int CONV>
static void qs_launch_render_scaled(const QsRenderPackOf<CONV> &pack, int n, int tiles, const int2 *status, int store,
		bool oriented, size_t smem, cudaStream_t st) {
	if (oriented) qs_launch_render_store<D, true, CONV>(pack, n, tiles, status, store, smem, st);
	else qs_launch_render_store<D, false, CONV>(pack, n, tiles, status, store, 0, st);
}

template <int D>
static cudaError_t qs_render_configure_d(void) {
	const void *k[7] = {(const void *)qs_render_async_kernel<QS_RENDER_HWC, D, true>,
			(const void *)qs_render_async_kernel<QS_RENDER_CHW, D, true>,
			(const void *)qs_render_async_kernel<QS_RENDER_GREY, D, true>,
			(const void *)qs_render_async_kernel<QS_RENDER_GREY, D, true, QS_CONV_L>,
			(const void *)qs_render_async_kernel<QS_RENDER_HWC, D, true, QS_CONV_CMYK_RGB>,
			(const void *)qs_render_async_kernel<QS_RENDER_CHW, D, true, QS_CONV_CMYK_RGB>,
			(const void *)qs_render_async_kernel<QS_RENDER_GREY, D, true, QS_CONV_CMYK_L>};
	for (int i = 0; i < 7; i++) {
		cudaError_t e = cudaFuncSetAttribute(k[i], cudaFuncAttributeMaxDynamicSharedMemorySize, QS_RT_TB_BYTES);
		if (e != cudaSuccess) return e;
	}
	return cudaSuccess;
}

cudaError_t qs_render_configure(void) {
	cudaError_t e = qs_render_configure_d<1>();
	if (e == cudaSuccess) e = qs_render_configure_d<2>();
	if (e == cudaSuccess) e = qs_render_configure_d<4>();
	if (e == cudaSuccess) e = qs_render_configure_d<8>();
	return e;
}

template <int CONV, class Img>
static cudaError_t qs_launch_render_pack(const Img *imgs, int n, int tiles, const int2 *status, int store,
		int scale_denom, cudaStream_t st) {
	constexpr int CAP = sizeof(QsRenderPackOf<CONV>::img) / sizeof(Img);
	if (n > CAP) return cudaErrorInvalidValue;
	QsRenderPackOf<CONV> pack;
	memcpy(pack.img, imgs, (size_t)n * sizeof(Img));
	if (n < CAP) memset(pack.img + n, 0, (size_t)(CAP - n) * sizeof(Img));
	bool oriented = false;
	size_t smem = 0;                                     /* the staging of the transposing orientations */
	for (int i = 0; i < n; i++) {
		if (imgs[i].orient < 1 || imgs[i].orient > 8) return cudaErrorInvalidValue;
		if (imgs[i].orient > 1) oriented = true;
		if (imgs[i].orient >= 5) smem = QS_RT_TB_BYTES;
	}
	switch (scale_denom) {
	case 1: qs_launch_render_scaled<1, CONV>(pack, n, tiles, status, store, oriented, smem, st); break;
	case 2: qs_launch_render_scaled<2, CONV>(pack, n, tiles, status, store, oriented, smem, st); break;
	case 4: qs_launch_render_scaled<4, CONV>(pack, n, tiles, status, store, oriented, smem, st); break;
	case 8: qs_launch_render_scaled<8, CONV>(pack, n, tiles, status, store, oriented, smem, st); break;
	default: return cudaErrorInvalidValue;
	}
	return cudaGetLastError();
}

cudaError_t qs_launch_render_async(const QsRenderImg *imgs, int n, int tiles, const int2 *status, int store,
		int scale_denom, cudaStream_t st, int conv) {
	if (tiles <= 0) return cudaSuccess;
	if (store != QS_RENDER_HWC && store != QS_RENDER_CHW && store != QS_RENDER_GREY) return cudaErrorInvalidValue;
	if (conv == QS_CONV_NONE) return qs_launch_render_pack<QS_CONV_NONE>(imgs, n, tiles, status, store, scale_denom, st);
	if (conv == QS_CONV_L && store == QS_RENDER_GREY)
		return qs_launch_render_pack<QS_CONV_L>(imgs, n, tiles, status, store, scale_denom, st);
	return cudaErrorInvalidValue;
}

cudaError_t qs_launch_render4_async(const QsRenderImg4 *imgs, int n, int tiles, int store, int conv, int scale_denom,
		cudaStream_t st) {
	if (tiles <= 0) return cudaSuccess;
	if (conv == QS_CONV_CMYK_RGB && (store == QS_RENDER_HWC || store == QS_RENDER_CHW))
		return qs_launch_render_pack<QS_CONV_CMYK_RGB>(imgs, n, tiles, NULL, store, scale_denom, st);
	if (conv == QS_CONV_CMYK_L && store == QS_RENDER_GREY)
		return qs_launch_render_pack<QS_CONV_CMYK_L>(imgs, n, tiles, NULL, store, scale_denom, st);
	return cudaErrorInvalidValue;
}

/* sample (x, y) of a host plane of `stride` samples per row */
struct QsHostPx {
	const uint8_t *s; int stride;
	__host__ __device__ int operator()(int x, int y) const { return s[(size_t)y * stride + x]; }
};

template <int D, class Img>
static void qs_render_host_d(const Img &im, int store, int conv) {
	constexpr int NC = sizeof(Img::coef) / sizeof(Img::coef[0]);
	const int nc = im.ncomp, W = im.width, H = im.height;
	std::vector<uint8_t> plane[NC];
	QsHostPx px[NC];
	int hs[NC], vs[NC], cw[NC], ch[NC];
	for (int c = 0; c < nc; c++) {
		bool up = false;
		if constexpr (NC == 3) up = c > 0 && im.up_mode == 1;
		const int k = up ? 0 : c, lss = D == 1 ? 3 : (im.lss >> (2 * k)) & 3, ss = 1 << lss;
		const int16_t *coef = im.coef[c];
		if constexpr (NC == 3) if (up) coef = im.coef_up[c - 1];
		hs[c] = im.hs[k]; vs[c] = im.vs[k]; cw[c] = im.cw[k]; ch[c] = im.ch[k];
		/* the blocks that hold the real samples (the render reads no others) */
		const int nbx = (cw[c] + ss - 1) >> lss, nby = (ch[c] + ss - 1) >> lss, stride = nbx * ss;
		plane[c].assign((size_t)stride * nby * ss, 0);
		for (int by = 0; by < nby; by++)
			for (int bx = 0; bx < nbx; bx++) {
				const int16_t *b = coef + ((size_t)by * im.wblk[k] + bx) * 64;
				int cf[64];
				for (int i = 0; i < 64; i++) cf[i] = b[i] * im.q[c][i];
				qs_idct_scaled(cf, ss, plane[c].data() + ((size_t)by * ss * stride + (size_t)bx * ss), stride);
			}
		px[c] = QsHostPx{plane[c].data(), stride};
	}
	const bool ycc = nc >= 3 && im.ycc;
	for (int oy = 0; oy < H; oy++)
		for (int ox = 0; ox < W; ox++) {
			const int y = qs_upsample_at<D != 8>(px[0], hs[0], vs[0], cw[0], ch[0], ox, oy);
			int c1 = y, c2 = y, c3 = 0;
			if (nc >= 3) {
				c1 = qs_upsample_at<D != 8>(px[1], hs[1], vs[1], cw[1], ch[1], ox, oy);
				c2 = qs_upsample_at<D != 8>(px[2], hs[2], vs[2], cw[2], ch[2], ox, oy);
			}
			if (nc == 4) c3 = qs_upsample_at<D != 8>(px[NC - 1], hs[NC - 1], vs[NC - 1], cw[NC - 1], ch[NC - 1], ox, oy);
			const uint32_t v = conv == QS_CONV_L ? qs_convert_pixel<QS_CONV_L>(y, c1, c2, c3, ycc) :
					conv == QS_CONV_CMYK_RGB ? qs_convert_pixel<QS_CONV_CMYK_RGB>(y, c1, c2, c3, ycc) :
					conv == QS_CONV_CMYK_L ? qs_convert_pixel<QS_CONV_CMYK_L>(y, c1, c2, c3, ycc) :
					qs_convert_pixel<QS_CONV_NONE>(y, c1, c2, c3, ycc);
			const size_t i = (size_t)oy * W + ox;
			if (store == QS_RENDER_HWC) for (int j = 0; j < 3; j++) im.out[3 * i + j] = (uint8_t)(v >> (8 * j));
			else for (int j = 0; j < (store == QS_RENDER_GREY ? 1 : 3); j++) im.out[(size_t)j * W * H + i] = (uint8_t)(v >> (8 * j));
		}
}

template <class Img>
static void qs_render_host_any(const Img &im, int store, int scale_denom, int conv) {
	switch (scale_denom) {
	case 1: qs_render_host_d<1>(im, store, conv); break;
	case 2: qs_render_host_d<2>(im, store, conv); break;
	case 4: qs_render_host_d<4>(im, store, conv); break;
	default: qs_render_host_d<8>(im, store, conv); break;
	}
}

void qs_render_host(const QsRenderImg *im, int store, int scale_denom, int conv) {
	qs_render_host_any(*im, store, scale_denom, conv);
}

void qs_render4_host(const QsRenderImg4 *im, int store, int scale_denom, int conv) {
	qs_render_host_any(*im, store, scale_denom, conv);
}

cudaError_t qs_launch_render_rgb(const uint8_t *const *planes, const int *strides, const int *cw, const int *ch,
		const int *hs, const int *vs, int ncomp, int width, int height, int ycc, uint8_t *rgb, cudaStream_t st) {
	QsRenderArgs a;
	for (int c = 0; c < 3; c++) {
		int k = c < ncomp ? c : 0;
		a.plane[c] = planes[k]; a.stride[c] = strides[k]; a.cw[c] = cw[k]; a.ch[c] = ch[k]; a.hs[c] = hs[k]; a.vs[c] = vs[k];
	}
	a.ncomp = ncomp; a.width = width; a.height = height; a.ycc = ycc;
	dim3 blk(32, 8), grd((width + 31) / 32, (height + 7) / 8);
	qs_render_rgb_kernel<<<grd, blk, 0, st>>>(a, rgb);
	return cudaGetLastError();
}

cudaError_t qs_store_jobs(QsJob *dst, const QsJob *jobs_host, int n, cudaStream_t st) {
	for (int off = 0; off < n; off += QS_JOB_PACK) {
		QsJobPack pack;
		int cnt = n - off < QS_JOB_PACK ? n - off : QS_JOB_PACK;
		memcpy(pack.j, jobs_host + off, (size_t)cnt * sizeof(QsJob));
		if (cnt < QS_JOB_PACK) memset(pack.j + cnt, 0, (size_t)(QS_JOB_PACK - cnt) * sizeof(QsJob));
		qs_store_jobs_kernel<<<1, QS_JOB_PACK, 0, st>>>(pack, dst + off, cnt);
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess) return e;
	}
	return cudaSuccess;
}

cudaError_t qs_copy_flags(const int *src_dev, int *dst_mapped, int n, cudaStream_t st) {
	qs_copy_flags_kernel<<<1, 128, 0, st>>>(src_dev, dst_mapped, n);
	return cudaGetLastError();
}

cudaError_t qs_store_quant(QsQuantDev *dst, const QsQuantDev *q_host, int n, cudaStream_t st) {
	for (int off = 0; off < n; off += QS_QUANT_PACK) {
		QsQuantPack pack;
		int cnt = n - off < QS_QUANT_PACK ? n - off : QS_QUANT_PACK;
		memcpy(pack.q, q_host + off, (size_t)cnt * sizeof(QsQuantDev));
		if (cnt < QS_QUANT_PACK) memset(pack.q + cnt, 0, (size_t)(QS_QUANT_PACK - cnt) * sizeof(QsQuantDev));
		qs_store_quant_kernel<<<1, 256, 0, st>>>(pack, dst + off, cnt);
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess) return e;
	}
	return cudaSuccess;
}

cudaError_t qs_launch_async_status(const QsStatusPack *p, int n, const int *flags, int2 *status, cudaStream_t st) {
	if (n <= 0) return cudaSuccess;
	qs_async_status_kernel<<<(n + 127) / 128, 128, 0, st>>>(*p, n, flags, status);
	return cudaGetLastError();
}
