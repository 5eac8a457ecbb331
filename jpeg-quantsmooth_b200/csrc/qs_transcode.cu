/*
 * qs_transcode.cu - jpegqs_cuda_transcode (include/jpegqs_cuda.h): one JPEG file in host memory to
 * the smoothed file the jpegqs tool writes, through the device decoder, run_async and the device
 * encoder on the context's stream.  Host code only: the kernels are those of qs_decode.cu,
 * qs_scans.cu, qs_kernels.cu and qs_encode.cu, reached through their public entry points.
 */
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "jpegqs_cuda.h"
#include "qs_common.h"

/* include/libjpegqs.h's JPEGQS_FLAGS_MASK and JPEGQS_ITER_MAX (that header needs <jpeglib.h>) */
#define QS_FLAGS_MASK 0x7f
#define QS_ITER_MAX 100

struct jpegqs_cuda_ctx;
void qs_ctx_decode_info(jpegqs_cuda_ctx *ctx, int *device, cudaStream_t *stream, int *sub_bytes);
void qs_ctx_decode_done(jpegqs_cuda_ctx *ctx, int launches, const char *err);
void **qs_ctx_transcode_state(jpegqs_cuda_ctx *ctx);
void qs_ctx_set_last_ms(jpegqs_cuda_ctx *ctx, float ms);
extern "C" int qs_route_plan(const uint8_t *data, size_t len, int copy, jpegqs_cuda_file_info *info, jpegqs_cuda_image *img,
		jpegqs_cuda_scan *scan, jpegqs_cuda_scan_rec *recs, int *nscans, jpegqs_cuda_jpeg_head *head,
		uint8_t **prefix, size_t *prefix_len, const char **reason);

/* the context's transcode buffers: device and pinned host memory, grow-only */
struct QsBuf { void *p; size_t cap; };
struct QsTranscode {
	QsBuf in_dev, coef_dev, ws_dev, out_dev;   /* file + prefix; coefficients + up-sampled chroma; the
	                                              workspace the three stages share; the output file */
	QsBuf in_host, out_host;                   /* pinned staging of the upload and the download */
	int32_t *small_dev, *small_host;           /* statuses and the length, 64 bytes */
	cudaEvent_t ev0, ev1;                      /* around run_async: jpegqs_cuda_last_device_ms */
	jpegqs_cuda_scan_rec recs[JPEGQS_MAX_SCANS];
};

/* layout of small_dev / small_host, in int32 words */
enum { SM_DECODE = 0, SM_RUN = 2, SM_LEN = 4, SM_ENCODE = 6, SM_WORDS = 16 };

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

void qs_transcode_release(void *state) {
	QsTranscode *t = (QsTranscode*)state;
	if (!t) return;
	cudaFree(t->in_dev.p); cudaFree(t->coef_dev.p); cudaFree(t->ws_dev.p); cudaFree(t->out_dev.p);
	cudaFree(t->small_dev);
	if (t->in_host.p) cudaFreeHost(t->in_host.p);
	if (t->out_host.p) cudaFreeHost(t->out_host.p);
	if (t->small_host) cudaFreeHost(t->small_host);
	if (t->ev0) cudaEventDestroy(t->ev0);
	if (t->ev1) cudaEventDestroy(t->ev1);
	delete t;
}

/* the stream is idle whenever these run: every call ends with a synchronisation */
static cudaError_t grow_dev(QsBuf *b, size_t need) {
	if (need <= b->cap) return cudaSuccess;
	if (b->p) cudaFree(b->p);
	b->p = NULL; b->cap = 0;
	size_t cap = align256(need + need / 8 + (1 << 16));
	cudaError_t e = cudaMalloc(&b->p, cap);
	if (e == cudaSuccess) b->cap = cap;
	return e;
}
static cudaError_t grow_host(QsBuf *b, size_t need) {
	if (need <= b->cap) return cudaSuccess;
	if (b->p) cudaFreeHost(b->p);
	b->p = NULL; b->cap = 0;
	size_t cap = align256(need + need / 8 + (1 << 16));
	cudaError_t e = cudaMallocHost(&b->p, cap);
	if (e == cudaSuccess) b->cap = cap;
	return e;
}

extern "C" void jpegqs_cuda_transcode_free(void *p) { free(p); }

extern "C" int jpegqs_cuda_transcode(jpegqs_cuda_ctx *ctx, const uint8_t *data, size_t len, int flags, int niter,
		int optimize, int copy, jpegqs_cuda_transcode_result *result) {
	char msg[512];
	if (!ctx) return JPEGQS_ERR_ARG;
	if (!data || !result) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_transcode: NULL argument"); return JPEGQS_ERR_ARG; }
	memset(result, 0, sizeof(*result));
	result->reason = "";
	if (copy < 0 || copy > 2) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_transcode: copy level outside 0..2"); return JPEGQS_ERR_ARG; }
	int device, sub_bytes; cudaStream_t st;
	qs_ctx_decode_info(ctx, &device, &st, &sub_bytes);
#define TK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	snprintf(msg, sizeof(msg), "%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
	free(prefix); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_CUDA; } } while (0)
#define TQ(call) do { int r_ = (call); if (r_ < 0) { free(prefix); return r_; } } while (0)
	uint8_t *prefix = NULL; size_t plen = 0;
	QsTranscode **slot = (QsTranscode**)qs_ctx_transcode_state(ctx);
	TK(cudaSetDevice(device));
	if (!*slot) {
		QsTranscode *t = new QsTranscode();
		memset(t, 0, sizeof(*t));
		*slot = t;
		TK(cudaMalloc(&t->small_dev, SM_WORDS * sizeof(int32_t)));
		TK(cudaMallocHost(&t->small_host, SM_WORDS * sizeof(int32_t)));
		TK(cudaEventCreate(&t->ev0)); TK(cudaEventCreate(&t->ev1));
	}
	QsTranscode *t = *slot;

	/* the route, and everything the stages need of the file, from one markers-only walk */
	jpegqs_cuda_image img; jpegqs_cuda_scan scan; jpegqs_cuda_jpeg_head head; int nscans = 0; const char *why;
	memset(&head, 0, sizeof(head));
	int route = qs_route_plan(data, len, copy, NULL, &img, &scan, t->recs, &nscans, &head, &prefix, &plen, &why);
	if (route < 0) {
		snprintf(msg, sizeof(msg), "jpegqs_cuda_transcode: %s", why);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (route != JPEGQS_ROUTE_DEVICE) { result->reason = why; return JPEGQS_TRANSCODE_FALLBACK; }

	/* do_quantsmooth's early return (csrc/do_quantsmooth.c): nothing to smooth and nothing to
	 * up-sample leaves the coefficients and the quant tables as read */
	const jpegqs_cuda_comp *c = img.comp;
	int need_downsample = (flags & (QS_JOINT_YUV | QS_UPSAMPLE_UV)) && img.is_ycbcr && img.ncomp >= 3 &&
			c[1].h_samp == 1 && c[1].v_samp == 1 && c[2].h_samp == 1 && c[2].v_samp == 1;
	int smooth = !((niter > QS_ITER_MAX ? QS_ITER_MAX : niter) <= 0 && !((flags & QS_UPSAMPLE_UV) && need_downsample));
	int can_up = smooth && need_downsample && (flags & QS_UPSAMPLE_UV) && (c[0].h_samp != 1 || c[0].v_samp != 1);
	int rflags = flags & QS_FLAGS_MASK;

	/* sizes: file | prefix; components | two luma-sized chroma arrays; one workspace; output */
	size_t data_off = align256(len), coef_bytes = 0, up_bytes = 0, ws = 0, w, cap;
	for (int k = 0; k < img.ncomp; k++) coef_bytes += align256((size_t)c[k].wblk * c[k].hblk * 128);
	if (can_up) up_bytes = 2 * align256((size_t)c[0].wblk * c[0].hblk * 128);
	if (!nscans) TQ(jpegqs_cuda_decode_workspace_bytes(1, &img, &scan, &len, &w));
	else { const jpegqs_cuda_scan_rec *r = t->recs; TQ(jpegqs_cuda_decode_scans_workspace_bytes(1, &img, &r, &nscans, &len, &w)); }
	ws = w;
	if (smooth) { TQ(jpegqs_cuda_async_workspace_bytes(1, &img, rflags, &w)); if (w > ws) ws = w; }
	TQ(jpegqs_cuda_encode_workspace_bytes(1, &img, optimize, &w)); if (w > ws) ws = w;
	TQ(jpegqs_cuda_encode_bound(&img, plen, &cap));
	TK(grow_dev(&t->in_dev, data_off + plen + 1));
	TK(grow_dev(&t->coef_dev, coef_bytes + up_bytes + 256));
	TK(grow_dev(&t->ws_dev, ws));
	TK(grow_dev(&t->out_dev, cap));
	TK(grow_host(&t->in_host, data_off + plen + 1));

	char *cp = (char*)t->coef_dev.p;
	for (int k = 0; k < img.ncomp; k++) { img.comp[k].coef = (int16_t*)cp; cp += align256((size_t)c[k].wblk * c[k].hblk * 128); }
	if (can_up) for (int k = 1; k <= 2; k++) { img.comp[k].coef_up = (int16_t*)cp; cp += up_bytes / 2; }
	uint8_t *in_dev = (uint8_t*)t->in_dev.p, *out_dev = (uint8_t*)t->out_dev.p;
	int32_t *sm = t->small_dev;
	head.prefix_dev = in_dev + data_off; head.prefix_len = (uint32_t)plen;

	memcpy(t->in_host.p, data, len);
	memcpy((char*)t->in_host.p + data_off, prefix, plen);
	free(prefix); prefix = NULL;
	TK(cudaMemcpyAsync(in_dev, t->in_host.p, data_off + plen, cudaMemcpyHostToDevice, st));
	if (!nscans) TQ(jpegqs_cuda_decode_async(ctx, 1, &img, &scan, &in_dev, &len, t->ws_dev.p, t->ws_dev.cap, sm + SM_DECODE, st));
	else {
		const jpegqs_cuda_scan_rec *r = t->recs; const uint8_t *d = in_dev;
		TQ(jpegqs_cuda_decode_scans_async(ctx, 1, &img, &r, &nscans, &d, &len, t->ws_dev.p, t->ws_dev.cap, sm + SM_DECODE, st));
	}
	const jpegqs_cuda_status *run_status = NULL;
	if (smooth) {
		TK(cudaEventRecord(t->ev0, st));
		TQ(jpegqs_cuda_run_async(ctx, 1, &img, rflags, niter, t->ws_dev.p, t->ws_dev.cap, (jpegqs_cuda_status*)(sm + SM_RUN), st));
		TK(cudaEventRecord(t->ev1, st));
		run_status = (const jpegqs_cuda_status*)(sm + SM_RUN);
	} else TK(cudaMemsetAsync(sm + SM_RUN, 0, 2 * sizeof(int32_t), st));
	TQ(jpegqs_cuda_encode_async(ctx, 1, &img, &head, optimize, run_status, &out_dev, &cap, (uint64_t*)(sm + SM_LEN),
			sm + SM_ENCODE, t->ws_dev.p, t->ws_dev.cap, st));
	TK(cudaMemcpyAsync(t->small_host, sm, SM_WORDS * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
	TK(cudaStreamSynchronize(st));

	const int32_t *h = t->small_host;
	uint64_t out_len; memcpy(&out_len, h + SM_LEN, sizeof(out_len));
	if (smooth) {
		float ms = 0;
		TK(cudaEventElapsedTime(&ms, t->ev0, t->ev1));
		qs_ctx_set_last_ms(ctx, ms);
	}
	result->smoothed = smooth; result->stop = h[SM_RUN]; result->upsampled = h[SM_RUN + 1];
	if (h[SM_DECODE]) { result->reason = "the device decoder flagged the data"; return JPEGQS_TRANSCODE_FALLBACK; }
	if (h[SM_ENCODE] & JPEGQS_ENCODE_RANGE) { result->reason = "a coefficient out of range for Huffman coding"; return JPEGQS_TRANSCODE_FALLBACK; }
	if (h[SM_ENCODE] || out_len > cap) {
		snprintf(msg, sizeof(msg), "jpegqs_cuda_transcode: encoder status %d, length %llu of %zu", (int)h[SM_ENCODE],
				(unsigned long long)out_len, cap);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_CUDA;
	}
	TK(grow_host(&t->out_host, out_len + 1));
	TK(cudaMemcpyAsync(t->out_host.p, out_dev, out_len, cudaMemcpyDeviceToHost, st));
	TK(cudaStreamSynchronize(st));
	result->data = (uint8_t*)malloc(out_len ? out_len : 1);
	if (!result->data) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_transcode: out of memory"); return JPEGQS_ERR_ARG; }
	memcpy(result->data, t->out_host.p, out_len);
	result->len = out_len;
	return JPEGQS_TRANSCODE_OK;
#undef TK
#undef TQ
}
