/*
 * qs_transcode.cu - jpegqs_cuda_transcode_batch and jpegqs_cuda_transcode (include/jpegqs_cuda.h):
 * JPEG files in host memory to the smoothed files the jpegqs tool writes, through the device
 * decoders, run_async and the device encoder on the context's stream, many files per launch.  The
 * decode, smoothing and encode kernels are those of qs_decode.cu, qs_scans.cu, qs_kernels.cu and
 * qs_encode.cu, reached through their public entry points; the one kernel here packs the encoded
 * files into one buffer so that a sub-batch comes back in one copy.
 * jpegqs_cuda_pixels_batch: the same files to the smoothed pixels the tool's --ppm writes, through
 * the same plans, sub-batches and decoder launches, the host reader, run_async and the fused render;
 * jpegqs_cuda_pixels_batch_resized adds qs_resize.cu's crop and resize after the render, and
 * jpegqs_cuda_pixels_batch_reduced qs_reduce.cu's reduce before the resize, and thumbnail's own scales;
 * jpegqs_cuda_pixels_batch_filtered qs_filter.cu's blurs after every other stage.
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "jpegqs_cuda.h"
#include "qs_common.h"
#include "qs_resize.h"
#include "qs_reduce.h"
#include "qs_filter.h"

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
int qs_render_takes(const jpegqs_cuda_image *im, int mode);           /* qs_cuda.cu */
int qs_render_images(jpegqs_cuda_ctx *ctx, int nimages, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_status *status_dev, int layout, int grey_store, int scale_denom, const int32_t *orient,
		uint8_t *const *out_dev, void *stream, int mode, const int32_t *color_space);

/* ---- the packing kernel -------------------------------------------------------------------------
 * After encode_async, file k of a sub-batch sits at the start of its bound-sized slot.  One launch
 * scans the lengths of the clean files (decoder status 0, encoder status 0, length within the slot)
 * and copies each of them to packed + off[k], off[k] = the exclusive sum of the preceding clean
 * lengths rounded up to 16 bytes, so that source (256-byte aligned slots) and destination both take
 * 16-byte vector copies and only a file's last partial vector is copied bytewise.  It also writes the
 * per-file record the host reads back: offset, length and the three status words.
 * Every block computes the scan of all files into shared memory (at most QS_PACK_MAX files, a few
 * microseconds of L2 reads), then takes 16 KB chunks of the concatenated output grid-stride: a chunk
 * finds its file by a binary search over the chunk counts. */
#define QS_PACK_THREADS 256
#define QS_PACK_MAX 1024                 /* files per sub-batch */
#define QS_PACK_CHUNK 16384              /* bytes per work item: four 16-byte vectors per thread */

struct QsPackDesc { uint64_t slot, cap; int32_t dec_idx, pad[3]; };          /* host -> device, 32 bytes */
struct QsPackRec { uint64_t off, len; int32_t decode, encode, stop, upsampled; };   /* device -> host, 32 bytes */

__global__ void __launch_bounds__(QS_PACK_THREADS) qs_pack_kernel(int n, const QsPackDesc *__restrict__ desc,
		const uint8_t *__restrict__ slots, const int32_t *__restrict__ dec, const jpegqs_cuda_status *__restrict__ run,
		const uint64_t *__restrict__ len, const int32_t *__restrict__ enc, QsPackRec *__restrict__ table,
		uint8_t *__restrict__ packed) {
	__shared__ uint64_t s_off[QS_PACK_MAX + 1];
	__shared__ uint32_t s_chk[QS_PACK_MAX + 1];
	__shared__ uint64_t w_off[QS_PACK_THREADS / 32];
	__shared__ uint32_t w_chk[QS_PACK_THREADS / 32];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint64_t carry_off = 0; uint32_t carry_chk = 0;
	for (int base = 0; base < n; base += QS_PACK_THREADS) {
		const int f = base + threadIdx.x;
		uint64_t L = 0; int32_t d = 0, e = 0;
		if (f < n) {
			L = len[f]; d = dec[desc[f].dec_idx]; e = enc[f];
			if (d || e || L > desc[f].cap) L = 0;
		}
		uint64_t a = (L + 15) & ~(uint64_t)15; uint32_t c = (uint32_t)((L + QS_PACK_CHUNK - 1) / QS_PACK_CHUNK);
		for (int s = 1; s < 32; s <<= 1) {                     /* inclusive warp scans */
			uint64_t ao = __shfl_up_sync(0xffffffffu, a, s); uint32_t co = __shfl_up_sync(0xffffffffu, c, s);
			if (lane >= s) { a += ao; c += co; }
		}
		if (lane == 31) { w_off[warp] = a; w_chk[warp] = c; }
		__syncthreads();
		uint64_t wa = 0, ta = 0; uint32_t wc = 0, tc = 0;
		for (int w = 0; w < QS_PACK_THREADS / 32; w++) {
			if (w < warp) { wa += w_off[w]; wc += w_chk[w]; }
			ta += w_off[w]; tc += w_chk[w];
		}
		if (f < n) {
			const uint64_t La = (L + 15) & ~(uint64_t)15;
			const uint32_t Lc = (uint32_t)((L + QS_PACK_CHUNK - 1) / QS_PACK_CHUNK);
			s_off[f] = carry_off + wa + a - La;
			s_chk[f] = carry_chk + wc + c - Lc;
			if (blockIdx.x == 0) {
				QsPackRec r; r.off = s_off[f]; r.len = len[f]; r.decode = d; r.encode = e;
				r.stop = run[f].stop; r.upsampled = run[f].upsampled;
				table[f] = r;
			}
		}
		carry_off += ta; carry_chk += tc;
		__syncthreads();                                        /* w_off / w_chk are reused */
	}
	if (threadIdx.x == 0) { s_off[n] = carry_off; s_chk[n] = carry_chk; }
	__syncthreads();
	const uint32_t total = s_chk[n];
	for (uint32_t c = blockIdx.x; c < total; c += gridDim.x) {
		/* the last file whose first chunk is <= c: it has chunks (s_chk[n] = total > c) */
		int lo = 0, hi = n - 1;
		while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (s_chk[mid] <= c) lo = mid; else hi = mid - 1; }
		const uint64_t start = (uint64_t)(c - s_chk[lo]) * QS_PACK_CHUNK, L = len[lo];
		const uint32_t bytes = (uint32_t)min((uint64_t)QS_PACK_CHUNK, L - start);
		const uint8_t *src = slots + desc[lo].slot + start;
		uint8_t *dst = packed + s_off[lo] + start;
		const uint4 *s4 = (const uint4*)src; uint4 *d4 = (uint4*)dst;
		const uint32_t nv = bytes >> 4;
#pragma unroll 4
		for (uint32_t i = threadIdx.x; i < nv; i += QS_PACK_THREADS) __stcs(d4 + i, __ldcs(s4 + i));
		if (threadIdx.x < (bytes & 15)) dst[(nv << 4) + threadIdx.x] = src[(nv << 4) + threadIdx.x];
	}
}

/* ---- the context's buffers: device and pinned host memory, grow-only ------------------------------ */
struct QsBuf { void *p; size_t cap; };
struct QsTranscode {
	QsBuf in_dev, coef_dev, ws_dev, out_dev;   /* descriptors + files + prefixes; coefficients + up-sampled
	                                              chroma; the workspace the three stages share, then the
	                                              packed files; the output slots (pixels: run statuses +
	                                              rendered pixels) */
	QsBuf stat_dev;                            /* per-file status words and the records of the packing kernel */
	QsBuf in_host, out_host, stat_host;        /* pinned staging of the upload and the two downloads */
	QsBuf hcoef_dev, hcoef_host;               /* pixels: the host-decoded files' coefficients and their staging */
	QsBuf rs_dev, rs_host;                     /* resized pixels: descriptors + weight tables, intermediates,
	                                              rendered pictures; the staging of the descriptors and tables */
	QsBuf jp_dev, jp_host;                     /* JPEG outputs: packing descriptors, lengths, statuses, records
	                                              and the encoder's output slots; the staging of descriptors
	                                              and records */
	QsBuf ft_dev, ft_host;                     /* filtered pixels: descriptors, then each file's picture before
	                                              the filter and two scratch pictures; the descriptors' staging */
	cudaEvent_t ev0, ev1;                      /* around run_async: jpegqs_cuda_last_device_ms */
	int sms;
	jpegqs_cuda_scan_rec recs[JPEGQS_MAX_SCANS];
};

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
static size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

void qs_transcode_release(void *state) {
	QsTranscode *t = (QsTranscode*)state;
	if (!t) return;
	cudaFree(t->in_dev.p); cudaFree(t->coef_dev.p); cudaFree(t->ws_dev.p); cudaFree(t->out_dev.p); cudaFree(t->stat_dev.p);
	cudaFree(t->hcoef_dev.p); cudaFree(t->rs_dev.p); cudaFree(t->jp_dev.p); cudaFree(t->ft_dev.p);
	if (t->ft_host.p) cudaFreeHost(t->ft_host.p);
	if (t->jp_host.p) cudaFreeHost(t->jp_host.p);
	if (t->in_host.p) cudaFreeHost(t->in_host.p);
	if (t->out_host.p) cudaFreeHost(t->out_host.p);
	if (t->stat_host.p) cudaFreeHost(t->stat_host.p);
	if (t->hcoef_host.p) cudaFreeHost(t->hcoef_host.p);
	if (t->rs_host.p) cudaFreeHost(t->rs_host.p);
	if (t->ev0) cudaEventDestroy(t->ev0);
	if (t->ev1) cudaEventDestroy(t->ev1);
	delete t;
}

/* the stream is idle whenever these run: every sub-batch ends with a synchronisation */
static cudaError_t grow_dev(QsBuf *b, size_t need) {
	if (need <= b->cap) return cudaSuccess;
	if (b->p) cudaFree(b->p);
	b->p = NULL; b->cap = 0;
	size_t cap = align256(need + need / 8 + (1 << 16));
	cudaError_t e = cudaMalloc(&b->p, cap);
	if (e == cudaSuccess) b->cap = cap;
	return e;
}
/* keep: leading bytes of the old contents carried over into a new allocation */
static cudaError_t grow_host(QsBuf *b, size_t need, size_t keep = 0) {
	if (need <= b->cap) return cudaSuccess;
	void *p = NULL;
	size_t cap = align256(need + need / 8 + (1 << 16));
	cudaError_t e = cudaMallocHost(&p, cap);
	if (e != cudaSuccess) return e;
	if (keep) memcpy(p, b->p, keep);
	if (b->p) cudaFreeHost(b->p);
	b->p = p; b->cap = cap;
	return cudaSuccess;
}

extern "C" void jpegqs_cuda_transcode_free(void *p) { free(p); }

/* One file as the markers-only walk planned it, and what it needs of each buffer. */
struct QsPlan {
	jpegqs_cuda_image img; jpegqs_cuda_scan scan; jpegqs_cuda_jpeg_head head;
	std::vector<jpegqs_cuda_scan_rec> recs;    /* empty: one sequential scan (decode_async) */
	uint8_t *prefix; size_t plen;
	int go;                                    /* the file takes part in the sub-batches */
	int host;                                  /* pixels: the host reader decodes it */
	int smooth, can_up;
	int out_w, out_h;                          /* pixels: the output picture's size */
	int orient, pic_w;                         /* pixels: the render's orientation (1..8), the rendered picture's width */
	int scale;                                 /* pixels: the render's scale denominator */
	int resized, reduced;                      /* pixels: the file goes through the resize; through the reduce first */
	int channels;                              /* pixels: 1 or 3, from the mode (the component count for mode 0) */
	size_t in_bytes, coef_bytes, up_bytes, cap, pix;
	size_t ws_dec, ws_run, ws_enc;             /* this file's share of each stage's workspace */
	size_t fixed, packed;                      /* its share of the buffers outside the workspace; of the packed output */
};

/* bytes a sub-batch of these files needs: each file's fixed share (the batch decides what that
 * holds), and the shared workspace - the largest of the decoders', run_async's and the encoder's and of
 * the packed output.  Each stage's workspace formula is a sum over files (run_async's constant is
 * counted per file here, so this bounds the exact group figure from above). */
struct QsNeed {
	size_t fixed, dec, run, enc, packed;
	size_t total() const { size_t w = dec; if (run > w) w = run; if (enc > w) w = enc; if (packed > w) w = packed; return fixed + w; }
	void add(const QsPlan &p) { fixed += p.fixed; dec += p.ws_dec; run += p.ws_run; enc += p.ws_enc; packed += p.packed; }
};

/* The context's batch state (created on first use), its device and stream. */
static int batch_state(jpegqs_cuda_ctx *ctx, cudaStream_t *st, QsTranscode **out) {
	char msg[256];
	int device, sub_bytes;
	cudaError_t e;
	qs_ctx_decode_info(ctx, &device, st, &sub_bytes);
	QsTranscode **slot = (QsTranscode**)qs_ctx_transcode_state(ctx);
	if ((e = cudaSetDevice(device)) != cudaSuccess) goto fail;
	if (!*slot) {
		QsTranscode *t = new QsTranscode();
		memset(t, 0, sizeof(*t));
		*slot = t;
		if ((e = cudaEventCreate(&t->ev0)) != cudaSuccess || (e = cudaEventCreate(&t->ev1)) != cudaSuccess ||
				(e = cudaDeviceGetAttribute(&t->sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) goto fail;
	}
	*out = *slot;
	return 0;
fail:
	snprintf(msg, sizeof(msg), "%s:%d: batch state: %s", __FILE__, __LINE__, cudaGetErrorString(e));
	qs_ctx_decode_done(ctx, 0, msg);
	return JPEGQS_ERR_CUDA;
}

/* File i's route from one markers-only walk (qs_route_plan): img for every file the reader takes; for a
 * DEVICE file its scans, the upload (file + prefix) and the decoder workspace; with prefix != 0 the
 * head and prefix of copy level `copy`.  *route: the route, or JPEGQS_ERR_ARG with *why the reader's
 * complaint.  Returns 0 or a negative error of the workspace formulas. */
static int plan_route(QsPlan &p, const uint8_t *data, size_t len, int copy, int prefix, jpegqs_cuda_scan_rec *recs,
		int *route, const char **why) {
	int nscans = 0;
	memset(&p.head, 0, sizeof(p.head));
	*route = qs_route_plan(data, len, copy, NULL, &p.img, &p.scan, recs, &nscans, prefix ? &p.head : NULL,
			prefix ? &p.prefix : NULL, prefix ? &p.plen : NULL, why);
	if (*route != JPEGQS_ROUTE_DEVICE) return 0;
	p.recs.assign(recs, recs + nscans);
	p.in_bytes = align256(len) + align256(p.plen);
	if (p.recs.empty()) return jpegqs_cuda_decode_workspace_bytes(1, &p.img, &p.scan, &len, &p.ws_dec);
	const jpegqs_cuda_scan_rec *r = p.recs.data();
	return jpegqs_cuda_decode_scans_workspace_bytes(1, &p.img, &r, &nscans, &len, &p.ws_dec);
}

/* do_quantsmooth's early return (csrc/do_quantsmooth.c): nothing to smooth and nothing to up-sample
 * leaves the coefficients and the quant tables as read.  Then the coefficient and up-sampled chroma
 * bytes and run_async's workspace share. */
static int plan_run(QsPlan &p, int flags, int niter) {
	const jpegqs_cuda_comp *c = p.img.comp;
	int need_downsample = (flags & (QS_JOINT_YUV | QS_UPSAMPLE_UV)) && p.img.is_ycbcr && p.img.ncomp >= 3 &&
			c[1].h_samp == 1 && c[1].v_samp == 1 && c[2].h_samp == 1 && c[2].v_samp == 1;
	p.smooth = !((niter > QS_ITER_MAX ? QS_ITER_MAX : niter) <= 0 && !((flags & QS_UPSAMPLE_UV) && need_downsample));
	p.can_up = p.smooth && need_downsample && (flags & QS_UPSAMPLE_UV) && (c[0].h_samp != 1 || c[0].v_samp != 1);
	p.coef_bytes = 0; p.up_bytes = 0;
	for (int k = 0; k < p.img.ncomp; k++) p.coef_bytes += align256((size_t)c[k].wblk * c[k].hblk * 128);
	if (p.can_up) p.up_bytes = 2 * align256((size_t)c[0].wblk * c[0].hblk * 128);
	p.ws_run = 0;
	if (p.smooth) return jpegqs_cuda_async_workspace_bytes(1, &p.img, flags & QS_FLAGS_MASK, &p.ws_run);
	return 0;
}

/* the budget: 0 = half of what is free on the device now plus what these buffers already hold */
static cudaError_t batch_budget(const QsTranscode *t, size_t max_device_bytes, size_t *budget) {
	*budget = max_device_bytes;
	if (max_device_bytes) return cudaSuccess;
	size_t fr = 0, tot = 0;
	cudaError_t e = cudaMemGetInfo(&fr, &tot);
	*budget = (fr + t->in_dev.cap + t->coef_dev.cap + t->ws_dev.cap + t->out_dev.cap + t->stat_dev.cap + t->hcoef_dev.cap +
			t->rs_dev.cap + t->jp_dev.cap + t->ft_dev.cap) / 2;
	return e;
}

/* the next sub-batch: consecutive files that go, from *i0 on, while their needs stay within the budget
 * (a file bigger than the budget goes alone), at most QS_PACK_MAX files; empty at the end */
static std::vector<int> next_group(const std::vector<QsPlan> &plans, int n, int *i0, size_t budget) {
	std::vector<int> files;
	QsNeed need = {0, 0, 0, 0, 0};
	int i = *i0;
	for (; i < n && (int)files.size() < QS_PACK_MAX; i++) {
		if (!plans[i].go) continue;
		QsNeed with = need; with.add(plans[i]);
		if (!files.empty() && with.total() > budget) break;
		need = with; files.push_back(i);
	}
	*i0 = i;
	return files;
}

/* One sub-batch: its files in the order of the later stages, their images, and the positions (in
 * that order) of the files each device decoder takes. */
struct QsGroup {
	std::vector<int> order;
	std::vector<jpegqs_cuda_image> eimg;
	std::vector<int> seq_k, scan_k;
	std::vector<const uint8_t*> data_dev;
	void set(const std::vector<QsPlan> &plans, const std::vector<int> &ord) {
		order = ord;
		const size_t m = ord.size();
		eimg.resize(m); data_dev.assign(m, NULL); seq_k.clear(); scan_k.clear();
		for (size_t k = 0; k < m; k++) {
			const QsPlan &p = plans[ord[k]];
			eimg[k] = p.img;
			if (!p.host) (p.recs.empty() ? seq_k : scan_k).push_back((int)k);
		}
	}
};

/* the exact workspace of the two decoders for the group's device-decoded files (the larger one) */
static int group_decode_ws(const QsGroup &g, const std::vector<QsPlan> &plans, const size_t *len, size_t *ws) {
	size_t w; int r;
	*ws = 0;
	if (!g.seq_k.empty()) {
		std::vector<jpegqs_cuda_image> im; std::vector<jpegqs_cuda_scan> sc; std::vector<size_t> ln;
		for (int k : g.seq_k) { im.push_back(g.eimg[k]); sc.push_back(plans[g.order[k]].scan); ln.push_back(len[g.order[k]]); }
		if ((r = jpegqs_cuda_decode_workspace_bytes((int)im.size(), im.data(), sc.data(), ln.data(), &w)) < 0) return r;
		if (w > *ws) *ws = w;
	}
	if (!g.scan_k.empty()) {
		std::vector<jpegqs_cuda_image> im; std::vector<const jpegqs_cuda_scan_rec*> sc; std::vector<int> ns; std::vector<size_t> ln;
		for (int k : g.scan_k) {
			const QsPlan &p = plans[g.order[k]];
			im.push_back(g.eimg[k]); sc.push_back(p.recs.data()); ns.push_back((int)p.recs.size()); ln.push_back(len[g.order[k]]);
		}
		if ((r = jpegqs_cuda_decode_scans_workspace_bytes((int)im.size(), im.data(), sc.data(), ns.data(), ln.data(), &w)) < 0) return r;
		if (w > *ws) *ws = w;
	}
	return 0;
}

/* the device-decoded files' bytes (file | prefix, each 256-byte aligned) into the pinned staging from
 * offset io on; records where each file will be on the device.  Returns the end offset. */
static size_t group_stage(QsGroup &g, const std::vector<QsPlan> &plans, const uint8_t *const *data, const size_t *len,
		uint8_t *in_host, const uint8_t *in_dev, size_t io) {
	for (size_t k = 0; k < g.order.size(); k++) {
		const QsPlan &p = plans[g.order[k]]; const size_t L = len[g.order[k]];
		if (p.host) continue;
		memcpy(in_host + io, data[g.order[k]], L);
		if (p.plen) memcpy(in_host + io + align256(L), p.prefix, p.plen);
		g.data_dev[k] = in_dev + io;
		io += p.in_bytes;
	}
	return io;
}

/* a component's coefficient arrays from cp on, 256-byte aligned; returns the next free byte */
static char *place_coefs(jpegqs_cuda_image &im, char *cp) {
	for (int q = 0; q < im.ncomp; q++) { im.comp[q].coef = (int16_t*)cp; cp += align256((size_t)im.comp[q].wblk * im.comp[q].hblk * 128); }
	return cp;
}
static char *place_up(jpegqs_cuda_image &im, const QsPlan &p, char *cp) {
	if (p.can_up) for (int q = 1; q <= 2; q++) { im.comp[q].coef_up = (int16_t*)cp; cp += p.up_bytes / 2; }
	return cp;
}

/* decode_async over the single-scan files and decode_scans_async over the others: statuses to dec[] in
 * that order */
static int group_decode(jpegqs_cuda_ctx *ctx, const QsGroup &g, const std::vector<QsPlan> &plans, const size_t *len,
		void *ws, size_t ws_cap, int32_t *dec, cudaStream_t st) {
	int r;
	if (!g.seq_k.empty()) {
		std::vector<jpegqs_cuda_image> im; std::vector<jpegqs_cuda_scan> sc; std::vector<const uint8_t*> dd; std::vector<size_t> ln;
		for (int k : g.seq_k) { im.push_back(g.eimg[k]); sc.push_back(plans[g.order[k]].scan); dd.push_back(g.data_dev[k]); ln.push_back(len[g.order[k]]); }
		if ((r = jpegqs_cuda_decode_async(ctx, (int)im.size(), im.data(), sc.data(), dd.data(), ln.data(), ws, ws_cap, dec, st)) < 0) return r;
	}
	if (!g.scan_k.empty()) {
		std::vector<jpegqs_cuda_image> im; std::vector<const jpegqs_cuda_scan_rec*> sc; std::vector<int> ns;
		std::vector<const uint8_t*> dd; std::vector<size_t> ln;
		for (int k : g.scan_k) {
			const QsPlan &p = plans[g.order[k]];
			im.push_back(g.eimg[k]); sc.push_back(p.recs.data()); ns.push_back((int)p.recs.size());
			dd.push_back(g.data_dev[k]); ln.push_back(len[g.order[k]]);
		}
		if ((r = jpegqs_cuda_decode_scans_async(ctx, (int)im.size(), im.data(), sc.data(), ns.data(), dd.data(), ln.data(),
				ws, ws_cap, dec + g.seq_k.size(), st)) < 0) return r;
	}
	return 0;
}

#define TK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	snprintf(msg, sizeof(msg), "%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
	qs_ctx_decode_done(ctx, 0, msg); ret = JPEGQS_ERR_CUDA; goto fail; } } while (0)
#define TQ(call) do { int r_ = (call); if (r_ < 0) { ret = r_; goto fail; } } while (0)

/* the batch; `who` names the entry point in error messages */
static int transcode_batch(jpegqs_cuda_ctx *ctx, const char *who, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int optimize, int copy, size_t max_device_bytes, int *rc, jpegqs_cuda_transcode_result *results) {
	char msg[512];
	cudaStream_t st;
	std::vector<QsPlan> plans((size_t)n);
	for (int i = 0; i < n; i++) plans[i].prefix = NULL;
	int ret = 0;
	{
	QsTranscode *t = NULL;
	TQ(batch_state(ctx, &st, &t));
	const int rflags = flags & QS_FLAGS_MASK;

	/* every file's route, and everything the stages need of it, from one markers-only walk */
	for (int i = 0; i < n; i++) {
		QsPlan &p = plans[i];
		int route; const char *why;
		TQ(plan_route(p, data[i], len[i], copy, 1, t->recs, &route, &why));
		if (route < 0) {
			if (n == 1) snprintf(msg, sizeof(msg), "%s: %s", who, why);
			else snprintf(msg, sizeof(msg), "%s: file %d: %s", who, i, why);
			qs_ctx_decode_done(ctx, 0, msg);
			rc[i] = JPEGQS_ERR_ARG; continue;
		}
		if (route != JPEGQS_ROUTE_DEVICE) { results[i].reason = why; rc[i] = JPEGQS_TRANSCODE_FALLBACK; continue; }
		rc[i] = JPEGQS_TRANSCODE_OK;
		TQ(plan_run(p, flags, niter));
		TQ(jpegqs_cuda_encode_workspace_bytes(1, &p.img, optimize, &p.ws_enc));
		TQ(jpegqs_cuda_encode_bound(&p.img, p.plen, &p.cap));
		/* file + prefix + descriptor, coefficients (+ up-sampled chroma), output slot */
		p.fixed = p.in_bytes + sizeof(QsPackDesc) + p.coef_bytes + p.up_bytes + align256(p.cap);
		p.packed = align16(p.cap);
		p.go = 1;
	}

	size_t budget;
	TK(batch_budget(t, max_device_bytes, &budget));

	/* sub-batches: consecutive device files while their needs stay within the budget */
	int i0 = 0;
	while (i0 < n) {
		std::vector<int> files = next_group(plans, n, &i0, budget);
		if (files.empty()) continue;
		const int m = (int)files.size();

		/* encode order: the files that smooth first, so run_async's status array is a prefix of the
		 * encoder's; decoder statuses: the single-scan files, then the others */
		std::vector<int> order; order.reserve(m);
		for (int f : files) if (plans[f].smooth) order.push_back(f);
		const int ms = (int)order.size();
		for (int f : files) if (!plans[f].smooth) order.push_back(f);
		QsGroup g; g.set(plans, order);
		std::vector<jpegqs_cuda_image> &eimg = g.eimg;
		std::vector<jpegqs_cuda_jpeg_head> heads(m);
		std::vector<uint8_t*> out_ptr(m);
		std::vector<size_t> caps(m);
		std::vector<QsPackDesc> desc(m);

		/* exact workspace of each stage for this group; the packed output shares the workspace */
		size_t ws = 0, w, in_total = align256((size_t)m * sizeof(QsPackDesc)), coef_total = 0, out_total = 0, packed = 0;
		TQ(group_decode_ws(g, plans, len, &ws));
		if (ms) { TQ(jpegqs_cuda_async_workspace_bytes(ms, eimg.data(), rflags, &w)); if (w > ws) ws = w; }
		TQ(jpegqs_cuda_encode_workspace_bytes(m, eimg.data(), optimize, &w)); if (w > ws) ws = w;
		for (int k = 0; k < m; k++) {
			const QsPlan &p = plans[order[k]];
			in_total += p.in_bytes; coef_total += p.coef_bytes + p.up_bytes; out_total += align256(p.cap); packed += align16(p.cap);
		}
		if (packed > ws) ws = packed;
		/* status words: lengths, run statuses, decoder statuses, encoder statuses, then the records */
		const size_t st_len = 0, st_run = align256(8 * (size_t)m), st_dec = st_run + align256(8 * (size_t)m),
				st_enc = st_dec + align256(4 * (size_t)m), st_tab = st_enc + align256(4 * (size_t)m),
				st_total = st_tab + (size_t)m * sizeof(QsPackRec);
		TK(grow_dev(&t->in_dev, in_total));
		TK(grow_dev(&t->coef_dev, coef_total + 256));
		TK(grow_dev(&t->ws_dev, ws));
		TK(grow_dev(&t->out_dev, out_total));
		TK(grow_dev(&t->stat_dev, st_total));
		TK(grow_host(&t->in_host, in_total));
		TK(grow_host(&t->stat_host, (size_t)m * sizeof(QsPackRec)));

		/* pointers, and the upload packed into the pinned staging: descriptors, then file | prefix */
		uint8_t *in_dev = (uint8_t*)t->in_dev.p, *in_host = (uint8_t*)t->in_host.p, *sd = (uint8_t*)t->stat_dev.p;
		char *cp = (char*)t->coef_dev.p;
		size_t io = align256((size_t)m * sizeof(QsPackDesc)), oo = 0;
		group_stage(g, plans, data, len, in_host, in_dev, io);
		for (int k = 0; k < m; k++) {
			QsPlan &p = plans[order[k]];
			cp = place_up(eimg[k], p, place_coefs(eimg[k], cp));
			heads[k] = p.head; heads[k].prefix_dev = g.data_dev[k] + align256(len[order[k]]); heads[k].prefix_len = (uint32_t)p.plen;
			out_ptr[k] = (uint8_t*)t->out_dev.p + oo; caps[k] = p.cap;
			memset(&desc[k], 0, sizeof(desc[k]));
			desc[k].slot = oo; desc[k].cap = p.cap;
			oo += align256(p.cap);
		}
		for (size_t q = 0; q < g.seq_k.size(); q++) desc[g.seq_k[q]].dec_idx = (int32_t)q;
		for (size_t q = 0; q < g.scan_k.size(); q++) desc[g.scan_k[q]].dec_idx = (int32_t)(g.seq_k.size() + q);
		memcpy(in_host, desc.data(), (size_t)m * sizeof(QsPackDesc));
		TK(cudaMemcpyAsync(in_dev, in_host, in_total, cudaMemcpyHostToDevice, st));

		int32_t *dec = (int32_t*)(sd + st_dec), *enc = (int32_t*)(sd + st_enc);
		jpegqs_cuda_status *run = (jpegqs_cuda_status*)(sd + st_run);
		uint64_t *lens = (uint64_t*)(sd + st_len);
		TQ(group_decode(ctx, g, plans, len, t->ws_dev.p, t->ws_dev.cap, dec, st));
		if (ms) {
			TK(cudaEventRecord(t->ev0, st));
			TQ(jpegqs_cuda_run_async(ctx, ms, eimg.data(), rflags, niter, t->ws_dev.p, t->ws_dev.cap, run, st));
			TK(cudaEventRecord(t->ev1, st));
		}
		if (ms < m) TK(cudaMemsetAsync(run + ms, 0, (size_t)(m - ms) * sizeof(jpegqs_cuda_status), st));
		/* files that did not smooth: run status 0, so the encoder writes them at their sampling */
		TQ(jpegqs_cuda_encode_async(ctx, m, eimg.data(), heads.data(), optimize, run, out_ptr.data(), caps.data(), lens,
				enc, t->ws_dev.p, t->ws_dev.cap, st));
		{
			size_t chunks = (packed + QS_PACK_CHUNK - 1) / QS_PACK_CHUNK, grid = 4 * (size_t)(t->sms > 0 ? t->sms : 1);
			if (chunks < grid) grid = chunks ? chunks : 1;
			qs_pack_kernel<<<(unsigned)grid, QS_PACK_THREADS, 0, st>>>(m, (const QsPackDesc*)in_dev, (const uint8_t*)t->out_dev.p,
					dec, run, lens, enc, (QsPackRec*)(sd + st_tab), (uint8_t*)t->ws_dev.p);
			TK(cudaGetLastError());
		}
		TK(cudaMemcpyAsync(t->stat_host.p, sd + st_tab, (size_t)m * sizeof(QsPackRec), cudaMemcpyDeviceToHost, st));
		TK(cudaStreamSynchronize(st));
		if (ms) {
			float ms_run = 0;
			TK(cudaEventElapsedTime(&ms_run, t->ev0, t->ev1));
			qs_ctx_set_last_ms(ctx, ms_run);
		}

		/* statuses; then exactly the packed bytes */
		const QsPackRec *rec = (const QsPackRec*)t->stat_host.p;
		size_t total = 0;
		for (int k = 0; k < m; k++) {
			const int f = order[k]; const QsPackRec &r = rec[k];
			jpegqs_cuda_transcode_result *res = &results[f];
			res->smoothed = plans[f].smooth; res->stop = r.stop; res->upsampled = r.upsampled;
			/* a flagged file's coefficients are unspecified (whatever its arrays held before): so is a
			 * run over them, and its status is not reported */
			if (r.decode) { res->stop = res->upsampled = 0; res->reason = "the device decoder flagged the data"; rc[f] = JPEGQS_TRANSCODE_FALLBACK; continue; }
			if (r.encode & JPEGQS_ENCODE_RANGE) { res->reason = "a coefficient out of range for Huffman coding"; rc[f] = JPEGQS_TRANSCODE_FALLBACK; continue; }
			if (r.encode || r.len > caps[k]) {
				snprintf(msg, sizeof(msg), "%s: encoder status %d, length %llu of %zu", who, (int)r.encode,
						(unsigned long long)r.len, caps[k]);
				qs_ctx_decode_done(ctx, 0, msg); ret = JPEGQS_ERR_CUDA; goto fail;
			}
			if (r.off + r.len > total) total = r.off + r.len;
		}
		if (total) {
			TK(grow_host(&t->out_host, total));
			TK(cudaMemcpyAsync(t->out_host.p, t->ws_dev.p, total, cudaMemcpyDeviceToHost, st));
			TK(cudaStreamSynchronize(st));
		}
		for (int k = 0; k < m; k++) {
			const int f = order[k]; const QsPackRec &r = rec[k];
			if (rc[f] != JPEGQS_TRANSCODE_OK) continue;
			results[f].data = (uint8_t*)malloc(r.len ? r.len : 1);
			if (!results[f].data) { snprintf(msg, sizeof(msg), "%s: out of memory", who); qs_ctx_decode_done(ctx, 0, msg); ret = JPEGQS_ERR_ARG; goto fail; }
			memcpy(results[f].data, (const uint8_t*)t->out_host.p + r.off, r.len);
			results[f].len = r.len;
		}
	}
	for (int i = 0; i < n; i++) free(plans[i].prefix);
	return 0;
	}
fail:
	for (int i = 0; i < n; i++) { free(plans[i].prefix); free(results[i].data); results[i].data = NULL; results[i].len = 0; }
	return ret;
}

extern "C" int jpegqs_cuda_transcode_batch(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int optimize, int copy, size_t max_device_bytes, int *rc, jpegqs_cuda_transcode_result *results) {
	static const char who[] = "jpegqs_cuda_transcode_batch";
	char msg[160];
	if (!ctx) return JPEGQS_ERR_ARG;
	if (n < 0) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_transcode_batch: negative file count"); return JPEGQS_ERR_ARG; }
	if (!n) return 0;
	if (!data || !len || !rc || !results) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_transcode_batch: NULL argument"); return JPEGQS_ERR_ARG; }
	for (int i = 0; i < n; i++) if (!data[i]) {
		snprintf(msg, sizeof(msg), "%s: file %d: NULL data", who, i);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	for (int i = 0; i < n; i++) { memset(&results[i], 0, sizeof(results[i])); results[i].reason = ""; rc[i] = 0; }
	if (copy < 0 || copy > 2) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_transcode_batch: copy level outside 0..2"); return JPEGQS_ERR_ARG; }
	return transcode_batch(ctx, who, n, data, len, flags, niter, optimize, copy, max_device_bytes, rc, results);
}

/* the batch of one */
extern "C" int jpegqs_cuda_transcode(jpegqs_cuda_ctx *ctx, const uint8_t *data, size_t len, int flags, int niter,
		int optimize, int copy, jpegqs_cuda_transcode_result *result) {
	if (!ctx) return JPEGQS_ERR_ARG;
	if (!data || !result) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_transcode: NULL argument"); return JPEGQS_ERR_ARG; }
	memset(result, 0, sizeof(*result));
	result->reason = "";
	if (copy < 0 || copy > 2) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_transcode: copy level outside 0..2"); return JPEGQS_ERR_ARG; }
	int rc = 0;
	int ret = transcode_batch(ctx, "jpegqs_cuda_transcode", 1, &data, &len, flags, niter, optimize, copy, 0, &rc, result);
	return ret < 0 ? ret : rc;
}

/* ---- JPEG files to smoothed pixels (jpegqs_cuda_pixels_batch) ------------------------------------- */
/* the host reader's decode of file f into the pinned staging at offset off; the warning count or
 * JPEGQS_ERR_ARG */
static int host_read(const QsPlan &p, const uint8_t *data, size_t len, uint8_t *staging, size_t off) {
	jpegqs_cuda_image im = p.img;
	place_coefs(im, (char*)staging + off);
	return jpegqs_cuda_jpeg_read(data, len, &im);
}

/* the JPEG outputs' device memory per sub-batch of m files (jp_dev): packing descriptors, lengths,
 * encoder statuses, zero decoder statuses, packing records, then the output slots */
struct QsJpegLayout {
	size_t desc, lens, enc, zero, rec, slots;
	void set(int m) {
		desc = 0; lens = align256(sizeof(QsPackDesc) * (size_t)m); enc = lens + align256(8 * (size_t)m);
		zero = enc + align256(4 * (size_t)m); rec = zero + align256(4 * (size_t)m); slots = rec + align256(sizeof(QsPackRec) * (size_t)m);
	}
};

/* the crop of a resize box in a pw x ph picture (all 0: the whole picture), or why it does not fit */
static const char *crop_of(const jpegqs_cuda_resize_box &b, int pw, int ph, int c[4]) {
	c[0] = b.left; c[1] = b.top; c[2] = b.right; c[3] = b.bottom;
	if (!c[0] && !c[1] && !c[2] && !c[3]) { c[2] = pw; c[3] = ph; }
	if (c[0] < 0 || c[1] < 0 || c[2] > pw || c[3] > ph) return "crop outside the picture";
	if (c[0] >= c[2] || c[1] >= c[3]) return "empty crop";
	return NULL;
}

/* boxes != NULL: each file's picture is cropped and resized (qs_resize.cu) with filter.  jp != NULL: the
 * pictures are written as JPEG files with these params (compress_async) into jout / jlen, and on_device
 * must be 0 (the pictures stay in the context's buffers).  orientation: NULL (1 for every file) or 0..8
 * per file, 0 for the file's own; the render writes the oriented picture, which the crop, the resize
 * and the compressor then take as it is.  mode: JPEGQS_PIXELS_*; the render converts, so every later stage
 * takes the converted picture's channels.  gap > 0: Pillow's reducing_gap, a reduce (qs_reduce.cu) before
 * the resize where its factor is above 1.  thumbnail: boxes hold bounds, each file is rendered at its
 * own draft scale and goes through the reduce and the resize only where Pillow's thumbnail does.
 * nfilters > 0: the earlier stages write each picture HWC into ft_dev, and filters (qs_filter.cu) take it
 * from there to the destination. */
static int pixels_batch(jpegqs_cuda_ctx *ctx, const char *who, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const int32_t *orientation, int mode, int on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results, const jpegqs_cuda_jpeg_params *jp = NULL, uint8_t **jout = NULL,
		size_t *jlen = NULL, int thumbnail = 0, double gap = 0.0, const jpegqs_cuda_image_filter *filters = NULL,
		int nfilters = 0) {
	char msg[512];
	cudaStream_t st;
	std::vector<QsPlan> plans((size_t)n);
	std::vector<QsResizePlan> rsp(boxes ? (size_t)n : 0);
	std::vector<QsReducePlan> rdp(boxes ? (size_t)n : 0);
	std::vector<size_t> pic(boxes ? (size_t)n : 0);  /* resized files: the rendered picture's bytes */
	const int loaded = orientation != NULL || mode != JPEGQS_PIXELS_AS_FILE;   /* thumbnail's draft does nothing */
	int ret = 0;
	{
	QsTranscode *t = NULL;
	TQ(batch_state(ctx, &st, &t));
	const int rflags = flags & QS_FLAGS_MASK;

	for (int i = 0; i < n; i++) {
		QsPlan &p = plans[i];
		int route; const char *why;
		p.prefix = NULL; p.plen = 0;
		TQ(plan_route(p, data[i], len[i], 0, 0, t->recs, &route, &why));
		if (route < 0) {
			snprintf(msg, sizeof(msg), "%s: file %d: %s", who, i, why);
			qs_ctx_decode_done(ctx, 0, msg);
			rc[i] = JPEGQS_ERR_ARG; continue;
		}
		if (!qs_render_takes(&p.img, mode)) { rc[i] = JPEGQS_ERR_UNSUPPORTED; continue; }
		p.channels = mode == JPEGQS_PIXELS_RGB ? 3 : mode == JPEGQS_PIXELS_L ? 1 : p.img.ncomp;
		/* the picture at scale 1 / scale_denom: ceil(width / d) x ceil(height / d) x channels, its axes
		 * swapped by orientations 5..8 */
		p.orient = orientation ? orientation[i] : 1;
		if (!p.orient && jpegqs_cuda_jpeg_orientation(data[i], len[i], &p.orient)) p.orient = 1;
		const int fw = (int)(p.orient >= 5 ? p.img.image_height : p.img.image_width);
		const int fh = (int)(p.orient >= 5 ? p.img.image_width : p.img.image_height);
		int tw = 0, th = 0;                         /* thumbnail: its size */
		p.scale = scale_denom;
		if (thumbnail) qs_thumbnail_geometry(fw, fh, boxes[i].width, boxes[i].height, gap, loaded, &p.scale, &tw, &th);
		const int sw = (int)((p.img.image_width + p.scale - 1) / p.scale);
		const int sh = (int)((p.img.image_height + p.scale - 1) / p.scale);
		const int pw = p.orient >= 5 ? sh : sw, ph = p.orient >= 5 ? sw : sh;
		p.pix = (size_t)pw * ph * p.channels;
		p.out_w = pw; p.out_h = ph; p.pic_w = pw;
		p.resized = boxes && (!thumbnail || pw != tw || ph != th);
		p.reduced = 0;
		if (p.resized) {
			const char *bad = NULL;
			if (thumbnail) {
				/* Image.resize(size, filter, box = draft's (0, 0, W / s, H / s), reducing_gap) */
				const double box[4] = {0.0, 0.0, gap > 0.0 && !loaded ? (double)fw / p.scale : (double)pw,
						gap > 0.0 && !loaded ? (double)fh / p.scale : (double)ph};
				bad = qs_reduced_plan(pw, ph, box, tw, th, filter, gap, rdp[i], rsp[i]);
			} else if (gap > 0.0) {
				/* crop, then Image.resize(size, filter, reducing_gap) of the crop */
				int c[4];
				bad = crop_of(boxes[i], pw, ph, c);
				if (!bad) {
					const double box[4] = {0.0, 0.0, (double)(c[2] - c[0]), (double)(c[3] - c[1])};
					bad = qs_reduced_plan(c[2] - c[0], c[3] - c[1], box, boxes[i].width, boxes[i].height, filter, gap, rdp[i], rsp[i]);
				}
				if (!bad && (rdp[i].fx > 1 || rdp[i].fy > 1)) { rdp[i].left += c[0]; rdp[i].top += c[1]; }
				else if (!bad) { rsp[i].left += c[0]; rsp[i].top += c[1]; }
			} else {
				bad = qs_resize_plan(pw, ph, boxes[i], filter, rsp[i]);
			}
			if (bad) {
				snprintf(msg, sizeof(msg), "%s: file %d: %s (picture %d x %d)", who, i, bad, pw, ph);
				qs_ctx_decode_done(ctx, 0, msg);
				rc[i] = JPEGQS_ERR_ARG; continue;
			}
			p.reduced = (thumbnail || gap > 0.0) && (rdp[i].fx > 1 || rdp[i].fy > 1);
			pic[i] = p.pix;
			p.out_w = rsp[i].out_w; p.out_h = rsp[i].out_h;
			p.pix = (size_t)p.out_w * p.out_h * p.channels;
		}
		p.host = route != JPEGQS_ROUTE_DEVICE;
		if (p.host) { p.in_bytes = 0; p.ws_dec = 0; results[i].host_decoded = 1; results[i].reason = why; }
		results[i].channels = p.channels;
		TQ(plan_run(p, flags, niter));
		/* file, coefficients (+ up-sampled chroma), the output pixels when they come back to the host;
		 * resized: also the rendered picture, the intermediate, the tables and the descriptor; reduced: the
		 * reduced picture and its descriptor */
		p.fixed = p.in_bytes + p.coef_bytes + p.up_bytes + (on_device ? 0 : align256(p.pix));
		if (p.resized)
			p.fixed += align256(pic[i]) + align256((size_t)rsp[i].mid_h * rsp[i].out_w * p.channels) +
					align256(rsp[i].tab.size() * sizeof(int32_t)) + align256(sizeof(QsResizeDesc));
		if (p.reduced)
			p.fixed += align256((size_t)rdp[i].out_w * rdp[i].out_h * p.channels) + align256(sizeof(QsReduceDesc));
		/* filtered: the picture before the filter, two scratch pictures and the pass descriptors */
		if (nfilters) p.fixed += 3 * align256(p.pix) + sizeof(QsFilterDesc) * QS_FILTER_MAX_STEPS * (size_t)nfilters;
		p.ws_enc = 0; p.packed = 0;
		if (jp) {
			/* JPEG: the compressor's workspace share (coefficients and encoder workspace, with the prefix's
			 * 256 bytes counted per file), its output slot, the packed copy and the per-file records */
			const jpegqs_cuda_pixels_in pin = { NULL, p.out_w, p.out_h, p.channels, (size_t)p.out_w * p.channels };
			TQ(jpegqs_cuda_compress_bound(&pin, jp, &p.cap));
			TQ(jpegqs_cuda_compress_workspace_bytes(1, &pin, jp, &p.ws_enc));
			p.packed = align16(p.cap);
			p.fixed += align256(p.cap) + 5 * 256;
		}
		p.go = 1;
	}

	size_t budget;
	TK(batch_budget(t, max_device_bytes, &budget));

	int i0 = 0;
	while (i0 < n) {
		std::vector<int> files = next_group(plans, n, &i0, budget);
		if (files.empty()) continue;
		const int m = (int)files.size();
		QsGroup g; g.set(plans, files);

		/* workspace: the decoders' and run_async's over every file that may smooth (a bound when a host
		 * read fails); device buffers: the uploaded files, the device-decoded files' coefficients and
		 * every file's up-sampled chroma, the decoder statuses */
		size_t ws = 0, w, in_total = 0, coef_total = 0;
		TQ(group_decode_ws(g, plans, len, &ws));
		{
			std::vector<jpegqs_cuda_image> sm;
			for (int k = 0; k < m; k++) if (plans[files[k]].smooth) sm.push_back(g.eimg[k]);
			if (!sm.empty()) { TQ(jpegqs_cuda_async_workspace_bytes((int)sm.size(), sm.data(), rflags, &w)); if (w > ws) ws = w; }
		}
		for (int f : files) in_total += plans[f].in_bytes, coef_total += (plans[f].host ? 0 : plans[f].coef_bytes) + plans[f].up_bytes;
		const int ndec = (int)(g.seq_k.size() + g.scan_k.size());
		/* JPEG: the compressor and encoder share the workspace once the render is done, then the packed
		 * files take it; jp_dev holds the slots and the small per-file arrays */
		QsJpegLayout jl;
		if (jp) {
			size_t cws = 256, packed = 0, slots = 0;
			for (int f : files) { cws += plans[f].ws_enc - 256; packed += plans[f].packed; slots += align256(plans[f].cap); }
			if (cws > ws) ws = cws;
			if (packed > ws) ws = packed;
			jl.set(m);
			TK(grow_dev(&t->jp_dev, jl.slots + slots));
			TK(grow_host(&t->jp_host, align256(sizeof(QsPackDesc) * (size_t)m) + sizeof(QsPackRec) * (size_t)m));
		}
		TK(grow_dev(&t->in_dev, in_total));
		TK(grow_dev(&t->coef_dev, coef_total + 256));
		TK(grow_dev(&t->ws_dev, ws));
		TK(grow_dev(&t->stat_dev, 4 * (size_t)m));
		TK(grow_host(&t->in_host, in_total));
		TK(grow_host(&t->stat_host, 4 * (size_t)m));

		/* 1-2: the files up, the decoders enqueued, their statuses down */
		group_stage(g, plans, data, len, (uint8_t*)t->in_host.p, (const uint8_t*)t->in_dev.p, 0);
		char *cp = (char*)t->coef_dev.p;
		for (int k = 0; k < m; k++) {
			const QsPlan &p = plans[files[k]];
			if (!p.host) cp = place_coefs(g.eimg[k], cp);
			cp = place_up(g.eimg[k], p, cp);
		}
		int32_t *dec = (int32_t*)t->stat_dev.p;
		if (in_total) TK(cudaMemcpyAsync(t->in_dev.p, t->in_host.p, in_total, cudaMemcpyHostToDevice, st));
		TQ(group_decode(ctx, g, plans, len, t->ws_dev.p, t->ws_dev.cap, dec, st));
		if (ndec) TK(cudaMemcpyAsync(t->stat_host.p, dec, 4 * (size_t)ndec, cudaMemcpyDeviceToHost, st));

		/* 3: the host-route files read while the device decodes, into the staging of the host-decoded
		 * coefficients (hoff: each file's offset there) */
		std::vector<size_t> hoff(m, 0);
		std::vector<char> alive(m, 1);
		size_t hb = 0;
		for (int k = 0; k < m; k++) if (plans[files[k]].host) { hoff[k] = hb; hb += plans[files[k]].coef_bytes; }
		TK(grow_host(&t->hcoef_host, hb));
		for (int k = 0; k < m; k++) {
			const int f = files[k];
			if (!plans[f].host) continue;
			int r = host_read(plans[f], data[f], len[f], (uint8_t*)t->hcoef_host.p, hoff[k]);
			if (r < 0) {
				snprintf(msg, sizeof(msg), "%s: file %d: %s", who, f, jpegqs_cuda_last_error(NULL));
				qs_ctx_decode_done(ctx, 0, msg);
				rc[f] = JPEGQS_ERR_ARG; alive[k] = 0; continue;
			}
			results[f].warnings = r;
		}
		TK(cudaStreamSynchronize(st));

		/* 4-5: a file the device decoder flagged is read again on the host, as the tool reads it */
		const int32_t *dh = (const int32_t*)t->stat_host.p;
		std::vector<int> dpos;                         /* decoder status index -> group position */
		for (int k : g.seq_k) dpos.push_back(k);
		for (int k : g.scan_k) dpos.push_back(k);
		for (int q = 0; q < ndec; q++) {
			if (!dh[q]) continue;
			const int k = dpos[q], f = files[k];
			const size_t keep = hb;
			hoff[k] = hb; hb += plans[f].coef_bytes;
			TK(grow_host(&t->hcoef_host, hb, keep));
			results[f].host_decoded = 1; results[f].reason = "the device decoder flagged the data";
			plans[f].host = 1;
			int r = host_read(plans[f], data[f], len[f], (uint8_t*)t->hcoef_host.p, hoff[k]);
			if (r < 0) {
				snprintf(msg, sizeof(msg), "%s: file %d: %s", who, f, jpegqs_cuda_last_error(NULL));
				qs_ctx_decode_done(ctx, 0, msg);
				rc[f] = JPEGQS_ERR_ARG; alive[k] = 0; continue;
			}
			results[f].warnings = r;
		}
		/* 6: the host-decoded coefficients up in one copy */
		if (hb) {
			TK(grow_dev(&t->hcoef_dev, hb));
			for (int k = 0; k < m; k++) if (plans[files[k]].host) place_coefs(g.eimg[k], (char*)t->hcoef_dev.p + hoff[k]);
			TK(cudaMemcpyAsync(t->hcoef_dev.p, t->hcoef_host.p, hb, cudaMemcpyHostToDevice, st));
		}

		/* 7: run_async over the files that smooth, then one render per render key (scale and layout; one
		 * key unless thumbnail).  Order the files that smooth by key, then by component count 3, 1, 4, and
		 * those that do not by key, then 4, 1, 3 - run_async's images are a prefix, each key's images are
		 * consecutive within each part, and each launch group's images (one store mode and conversion) are
		 * consecutive, so with one key the render takes at most five launches per 60 images (three without
		 * 4-component files) */
		std::vector<int> rk;                           /* render order -> group position */
		static const int kinds[6] = {3, 1, 4, 4, 1, 3};
		auto rkey = [&](const QsPlan &p) { return p.scale * 2 + (p.resized || nfilters ? JPEGQS_RENDER_HWC : layout); };
		for (int pass = 0; pass < 6; pass += 3)
			for (int key = 2; key <= 17; key++)
				for (int q = pass; q < pass + 3; q++)
					for (int k = 0; k < m; k++) {
						const QsPlan &p = plans[files[k]];
						if (alive[k] && p.smooth == (pass < 3) && p.img.ncomp == kinds[q] && rkey(p) == key) rk.push_back(k);
					}
		const int nr = (int)rk.size();
		int ms = 0;
		std::vector<jpegqs_cuda_image> rimg(nr);
		for (int j = 0; j < nr; j++) { rimg[j] = g.eimg[rk[j]]; if (plans[files[rk[j]]].smooth) ms++; }
		const size_t st_bytes = align256(sizeof(jpegqs_cuda_status) * (size_t)(nr ? nr : 1));
		std::vector<size_t> poff(nr);
		size_t pix_total = st_bytes;
		for (int j = 0; j < nr; j++) { poff[j] = pix_total; if (!on_device) pix_total += align256(plans[files[rk[j]]].pix); }
		const size_t down = jp ? st_bytes : pix_total;  /* JPEG: the pictures stay on the device */
		TK(grow_dev(&t->out_dev, pix_total));
		TK(grow_host(&t->out_host, down));
		jpegqs_cuda_status *run = (jpegqs_cuda_status*)t->out_dev.p;
		std::vector<uint8_t*> outs(nr);
		for (int j = 0; j < nr; j++) outs[j] = on_device ? out[files[rk[j]]] : (uint8_t*)t->out_dev.p + poff[j];
		/* filtered: the passes' descriptors (one upload from ft_host), then per file the picture the earlier
		 * stages write (outs from here on) and two scratch pictures; the last pass writes the destination */
		std::vector<QsFilterLaunch> flaunch;
		if (nfilters && nr) {
			std::vector<QsFilterPic> fp(nr);
			std::vector<QsFilterDesc> fdesc;
			size_t fo = align256(sizeof(QsFilterDesc) * QS_FILTER_MAX_STEPS * (size_t)nfilters * nr), all = fo;
			for (int j = 0; j < nr; j++) all += 3 * align256(plans[files[rk[j]]].pix);
			TK(grow_dev(&t->ft_dev, all));
			uint8_t *fd = (uint8_t*)t->ft_dev.p;
			for (int j = 0; j < nr; j++) {
				const QsPlan &p = plans[files[rk[j]]];
				const size_t a = align256(p.pix);
				fp[j].in = fd + fo; fp[j].a = fd + fo + a; fp[j].b = fd + fo + 2 * a; fp[j].out = outs[j];
				fp[j].w = p.out_w; fp[j].h = p.out_h; fp[j].ch = p.channels; fp[j].chw = layout == JPEGQS_RENDER_CHW;
				outs[j] = fp[j].in;
				fo += 3 * a;
			}
			qs_filter_plan(filters, nfilters, fp.data(), nr, fdesc, flaunch);
			TK(grow_host(&t->ft_host, sizeof(QsFilterDesc) * fdesc.size()));
			memcpy(t->ft_host.p, fdesc.data(), sizeof(QsFilterDesc) * fdesc.size());
			TK(cudaMemcpyAsync(fd, t->ft_host.p, sizeof(QsFilterDesc) * fdesc.size(), cudaMemcpyHostToDevice, st));
		}
		/* resized: the render writes each picture into rs_dev, which holds the resize descriptors, the
		 * reduce descriptors and the tables (one upload from rs_host), then the intermediates, then the
		 * pictures, then the reduced pictures; the reduce writes those, the resize writes outs */
		std::vector<int> rsj, rdj;                     /* render positions of the resized and the reduced files */
		for (int j = 0; j < nr; j++) {
			if (plans[files[rk[j]]].resized) rsj.push_back(j);
			if (plans[files[rk[j]]].reduced) rdj.push_back(j);
		}
		const int nrs = (int)rsj.size(), nrd = (int)rdj.size();
		uint32_t hblocks = 0, vblocks = 0, rblocks = 0;
		const size_t rdo = align256(sizeof(QsResizeDesc) * (size_t)nrs);
		if (nrs) {
			size_t up = rdo + align256(sizeof(QsReduceDesc) * (size_t)nrd), all;
			std::vector<size_t> toff(nrs), moff(nrs), qoff(nrs), roff(nrs);
			for (int q = 0; q < nrs; q++) { toff[q] = up; up += align256(rsp[files[rk[rsj[q]]]].tab.size() * sizeof(int32_t)); }
			all = up;
			for (int q = 0; q < nrs; q++) {
				const QsResizePlan &r = rsp[files[rk[rsj[q]]]];
				moff[q] = all; all += align256((size_t)r.mid_h * r.out_w * plans[files[rk[rsj[q]]]].channels);
			}
			for (int q = 0; q < nrs; q++) { qoff[q] = all; all += align256(pic[files[rk[rsj[q]]]]); }
			for (int q = 0; q < nrs; q++) {
				const int f = files[rk[rsj[q]]];
				roff[q] = all;
				if (plans[f].reduced) all += align256((size_t)rdp[f].out_w * rdp[f].out_h * plans[f].channels);
			}
			TK(grow_dev(&t->rs_dev, all));
			TK(grow_host(&t->rs_host, up));
			uint8_t *rd = (uint8_t*)t->rs_dev.p, *rh = (uint8_t*)t->rs_host.p;
			QsResizeDesc *desc = (QsResizeDesc*)rh;
			QsReduceDesc *rdesc = (QsReduceDesc*)(rh + rdo);
			int nq = 0;
			for (int q = 0; q < nrs; q++) {
				const int j = rsj[q], f = files[rk[j]];
				const QsResizePlan &r = rsp[f];
				const QsPlan &p = plans[f];
				qs_resize_desc(r, p.reduced ? rdp[f].out_w : p.pic_w, p.channels, layout == JPEGQS_RENDER_CHW && !nfilters, desc[q]);
				memcpy(rh + toff[q], r.tab.data(), r.tab.size() * sizeof(int32_t));
				desc[q].src = rd + (p.reduced ? roff[q] : qoff[q]); desc[q].mid = rd + moff[q]; desc[q].out = outs[j];
				desc[q].tab = (const int32_t*)(rd + toff[q]);
				if (p.reduced) {
					qs_reduce_desc(rdp[f], p.pic_w, p.channels, rdesc[nq]);
					rdesc[nq].src = rd + qoff[q]; rdesc[nq].out = rd + roff[q];
					nq++;
				}
				outs[j] = rd + qoff[q];
			}
			qs_resize_number(desc, nrs, &hblocks, &vblocks);
			rblocks = qs_reduce_number(rdesc, nrd);
			TK(cudaMemcpyAsync(rd, rh, up, cudaMemcpyHostToDevice, st));
		}
		if (ms) {
			TK(cudaEventRecord(t->ev0, st));
			TQ(jpegqs_cuda_run_async(ctx, ms, rimg.data(), rflags, niter, t->ws_dev.p, t->ws_dev.cap, run, st));
			TK(cudaEventRecord(t->ev1, st));
		}
		if (ms < nr) TK(cudaMemsetAsync(run + ms, 0, (size_t)(nr - ms) * sizeof(jpegqs_cuda_status), st));
		std::vector<int32_t> ro(nr), rcs(nr);
		for (int j = 0; j < nr; j++) { ro[j] = plans[files[rk[j]]].orient; rcs[j] = plans[files[rk[j]]].scan.jpeg_color_space; }
		for (int j0 = 0, j1; j0 < nr; j0 = j1) {
			const QsPlan &p0 = plans[files[rk[j0]]];
			for (j1 = j0 + 1; j1 < nr && rkey(plans[files[rk[j1]]]) == rkey(p0); j1++) {}
			TQ(qs_render_images(ctx, j1 - j0, rimg.data() + j0, run + j0, p0.resized || nfilters ? JPEGQS_RENDER_HWC : layout, 1, p0.scale,
					ro.data() + j0, outs.data() + j0, st, mode, mode ? rcs.data() + j0 : NULL));
		}
		if (nrd) TK(qs_launch_reduce((const QsReduceDesc*)((uint8_t*)t->rs_dev.p + rdo), nrd, rblocks, st));
		if (nrs) TK(qs_launch_resize((const QsResizeDesc*)t->rs_dev.p, nrs, hblocks, vblocks, st));
		if (!flaunch.empty()) TK(qs_filter_enqueue(flaunch, (const QsFilterDesc*)t->ft_dev.p, st));
		/* JPEG: compress_async over the pictures into the slots, then the packing kernel into the
		 * workspace, its records back */
		uint8_t *jd = (uint8_t*)t->jp_dev.p, *jh = (uint8_t*)t->jp_host.p;
		const size_t jh_rec = align256(sizeof(QsPackDesc) * (size_t)m);
		size_t packed = 0;
		if (jp && nr) {
			std::vector<jpegqs_cuda_pixels_in> pin(nr);
			std::vector<uint8_t*> slot(nr);
			std::vector<size_t> cap(nr);
			QsPackDesc *pd = (QsPackDesc*)jh;
			size_t so = 0;
			for (int j = 0; j < nr; j++) {
				const QsPlan &p = plans[files[rk[j]]];
				pin[j].pixels_dev = (const uint8_t*)t->out_dev.p + poff[j];
				pin[j].width = p.out_w; pin[j].height = p.out_h; pin[j].channels = p.channels;
				pin[j].row_bytes = (size_t)p.out_w * p.channels;
				slot[j] = jd + jl.slots + so; cap[j] = p.cap;
				memset(&pd[j], 0, sizeof(pd[j]));
				pd[j].slot = so; pd[j].cap = p.cap; pd[j].dec_idx = j;
				so += align256(p.cap); packed += align16(p.cap);
			}
			TK(cudaMemcpyAsync(jd + jl.desc, jh, sizeof(QsPackDesc) * (size_t)nr, cudaMemcpyHostToDevice, st));
			TK(cudaMemsetAsync(jd + jl.zero, 0, 4 * (size_t)nr, st));
			TQ(jpegqs_cuda_compress_async(ctx, nr, pin.data(), jp, slot.data(), cap.data(), (uint64_t*)(jd + jl.lens),
					(int32_t*)(jd + jl.enc), t->ws_dev.p, t->ws_dev.cap, st));
			size_t chunks = (packed + QS_PACK_CHUNK - 1) / QS_PACK_CHUNK, grid = 4 * (size_t)(t->sms > 0 ? t->sms : 1);
			if (chunks < grid) grid = chunks ? chunks : 1;
			qs_pack_kernel<<<(unsigned)grid, QS_PACK_THREADS, 0, st>>>(nr, (const QsPackDesc*)(jd + jl.desc), jd + jl.slots,
					(const int32_t*)(jd + jl.zero), run, (const uint64_t*)(jd + jl.lens), (const int32_t*)(jd + jl.enc),
					(QsPackRec*)(jd + jl.rec), (uint8_t*)t->ws_dev.p);
			TK(cudaGetLastError());
			TK(cudaMemcpyAsync(jh + jh_rec, jd + jl.rec, sizeof(QsPackRec) * (size_t)nr, cudaMemcpyDeviceToHost, st));
		}
		/* the run statuses, and the pixels in the same copy when they come back to the host */
		if (nr) TK(cudaMemcpyAsync(t->out_host.p, t->out_dev.p, down, cudaMemcpyDeviceToHost, st));
		TK(cudaStreamSynchronize(st));
		if (ms) {
			float ms_run = 0;
			TK(cudaEventElapsedTime(&ms_run, t->ev0, t->ev1));
			qs_ctx_set_last_ms(ctx, ms_run);
		}
		const jpegqs_cuda_status *rs = (const jpegqs_cuda_status*)t->out_host.p;
		for (int j = 0; j < nr; j++) {
			const int f = files[rk[j]];
			results[f].smoothed = plans[f].smooth; results[f].stop = rs[j].stop; results[f].upsampled = rs[j].upsampled;
			if (!on_device && !jp) memcpy(out[f], (const uint8_t*)t->out_host.p + poff[j], plans[f].pix);
		}
		if (jp && nr) {
			/* every file is clean (8-bit samples cannot make RANGE, the slots hold the bound): exactly the
			 * packed bytes back */
			const QsPackRec *rec = (const QsPackRec*)(jh + jh_rec);
			size_t total = 0;
			for (int j = 0; j < nr; j++) {
				if (rec[j].encode || rec[j].len > plans[files[rk[j]]].cap) {
					snprintf(msg, sizeof(msg), "%s: encoder status %d, length %llu of %zu", who, (int)rec[j].encode,
							(unsigned long long)rec[j].len, plans[files[rk[j]]].cap);
					qs_ctx_decode_done(ctx, 0, msg); ret = JPEGQS_ERR_CUDA; goto fail;
				}
				if (rec[j].off + rec[j].len > total) total = rec[j].off + rec[j].len;
			}
			TK(grow_host(&t->out_host, total));
			TK(cudaMemcpyAsync(t->out_host.p, t->ws_dev.p, total, cudaMemcpyDeviceToHost, st));
			TK(cudaStreamSynchronize(st));
			for (int j = 0; j < nr; j++) {
				const int f = files[rk[j]];
				jout[f] = (uint8_t*)malloc(rec[j].len);
				if (!jout[f]) { snprintf(msg, sizeof(msg), "%s: out of memory", who); qs_ctx_decode_done(ctx, 0, msg); ret = JPEGQS_ERR_ARG; goto fail; }
				memcpy(jout[f], (const uint8_t*)t->out_host.p + rec[j].off, rec[j].len);
				jlen[f] = rec[j].len;
			}
		}
	}
	return 0;
	}
fail:
	if (jout) for (int i = 0; i < n; i++) { free(jout[i]); jout[i] = NULL; jlen[i] = 0; }
	return ret;
}
#undef TK
#undef TQ

/* resize != 0: jpegqs_cuda_pixels_batch_resized, with filter and boxes */
/* an orientation array's check: NULL, or 0..8 per file */
static int orientation_ok(jpegqs_cuda_ctx *ctx, const char *who, int n, const int32_t *orientation) {
	char msg[200];
	for (int i = 0; orientation && i < n; i++) if (orientation[i] < 0 || orientation[i] > 8) {
		snprintf(msg, sizeof(msg), "%s: file %d: orientation %d outside 0..8", who, i, (int)orientation[i]);
		qs_ctx_decode_done(ctx, 0, msg); return 0;
	}
	return 1;
}

/* a colour mode's check: JPEGQS_PIXELS_AS_FILE, _RGB or _L */
static int mode_ok(jpegqs_cuda_ctx *ctx, const char *who, int mode) {
	if (mode == JPEGQS_PIXELS_AS_FILE || mode == JPEGQS_PIXELS_RGB || mode == JPEGQS_PIXELS_L) return 1;
	char msg[200];
	snprintf(msg, sizeof(msg), "%s: mode %d: expected 0 (as the file), 1 (RGB) or 2 (L)", who, mode);
	qs_ctx_decode_done(ctx, 0, msg);
	return 0;
}

/* reducing_gap and thumbnail's checks: gap 0 (None) or finite and at least 1; with thumbnail, boxes that
 * hold only bounds and scale_denom 1 */
static int reduced_ok(jpegqs_cuda_ctx *ctx, const char *who, int n, const jpegqs_cuda_resize_box *boxes, int scale_denom,
		int thumbnail, double gap) {
	char msg[200];
	const char *bad = !(gap == 0.0 || (isfinite(gap) && gap >= 1.0)) ? "reducing_gap must be 0 (None) or a finite value of at least 1.0" :
			thumbnail != 0 && thumbnail != 1 ? "thumbnail must be 0 or 1" :
			thumbnail && !boxes ? "boxes NULL" : thumbnail && scale_denom != 1 ? "scale_denom must be 1 with thumbnail" : NULL;
	for (int i = 0; i < n && !bad && thumbnail; i++)
		if (boxes[i].left || boxes[i].top || boxes[i].right || boxes[i].bottom) {
			snprintf(msg, sizeof(msg), "%s: file %d: a thumbnail box has no crop (left..bottom must be 0)", who, i);
			qs_ctx_decode_done(ctx, 0, msg); return 0;
		}
	if (!bad) return 1;
	snprintf(msg, sizeof(msg), "%s: %s", who, bad);
	qs_ctx_decode_done(ctx, 0, msg);
	return 0;
}

/* the filters' check: nfilters 0..64, each one qs_filter_check takes */
static int filters_ok(jpegqs_cuda_ctx *ctx, const char *who, const jpegqs_cuda_image_filter *filters, int nfilters) {
	char msg[240];
	const char *bad = nfilters < 0 || nfilters > 64 ? "nfilters outside 0..64" : nfilters && !filters ? "filters NULL" : NULL;
	int k = 0;
	for (; k < nfilters && !bad; k++) bad = qs_filter_check(filters[k]);
	if (!bad) return 1;
	if (k) snprintf(msg, sizeof(msg), "%s: filter %d: %s", who, k - 1, bad);
	else snprintf(msg, sizeof(msg), "%s: %s", who, bad);
	qs_ctx_decode_done(ctx, 0, msg);
	return 0;
}

static int pixels_entry(jpegqs_cuda_ctx *ctx, const char *who, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int resize, int filter, const jpegqs_cuda_resize_box *boxes,
		int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		const int32_t *orientation = NULL, int mode = JPEGQS_PIXELS_AS_FILE, int thumbnail = 0, double gap = 0.0,
		const jpegqs_cuda_image_filter *filters = NULL, int nfilters = 0) {
	char msg[200];
	if (!ctx) return JPEGQS_ERR_ARG;
	if (n < 0) { snprintf(msg, sizeof(msg), "%s: negative file count", who); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
	if (!n) return 0;
	if (!data || !len || !out || !rc || !results) { snprintf(msg, sizeof(msg), "%s: NULL argument", who); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
	for (int i = 0; i < n; i++) if (!data[i] || !out[i]) {
		snprintf(msg, sizeof(msg), "%s: file %d: NULL %s", who, i, data[i] ? "output" : "data");
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (layout != JPEGQS_RENDER_HWC && layout != JPEGQS_RENDER_CHW) { snprintf(msg, sizeof(msg), "%s: unknown layout", who); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
	if (scale_denom != 1 && scale_denom != 2 && scale_denom != 4 && scale_denom != 8) {
		snprintf(msg, sizeof(msg), "%s: scale_denom must be 1, 2, 4 or 8", who); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (out_on_device != 0 && out_on_device != 1) {
		snprintf(msg, sizeof(msg), "%s: out_on_device must be 0 or 1", who); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (resize) {
		if (!boxes) { snprintf(msg, sizeof(msg), "%s: boxes NULL", who); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
		if (!qs_resize_filter_ok(filter)) {
			snprintf(msg, sizeof(msg), "%s: filter %d: expected LANCZOS (1), BILINEAR (2), BICUBIC (3), BOX (4) or HAMMING (5)", who, filter);
			qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
		}
		for (int i = 0; i < n; i++) if (boxes[i].width < 1 || boxes[i].width > 65535 || boxes[i].height < 1 || boxes[i].height > 65535) {
			snprintf(msg, sizeof(msg), "%s: file %d: output size %d x %d outside 1..65535", who, i, boxes[i].width, boxes[i].height);
			qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
		}
	}
	if (!orientation_ok(ctx, who, n, orientation) || !mode_ok(ctx, who, mode) ||
			!reduced_ok(ctx, who, n, boxes, scale_denom, thumbnail, gap) || !filters_ok(ctx, who, filters, nfilters))
		return JPEGQS_ERR_ARG;
	for (int i = 0; i < n; i++) { memset(&results[i], 0, sizeof(results[i])); results[i].reason = ""; rc[i] = 0; }
	return pixels_batch(ctx, who, n, data, len, flags, niter, layout, scale_denom, filter, resize ? boxes : NULL, orientation,
			mode, out_on_device, out, max_device_bytes, rc, results, NULL, NULL, NULL, thumbnail, gap, filters, nfilters);
}

extern "C" int jpegqs_cuda_pixels_batch_filtered(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const int32_t *orientation, int mode, int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results, int thumbnail, double reducing_gap, const jpegqs_cuda_image_filter *filters,
		int nfilters) {
	return pixels_entry(ctx, "jpegqs_cuda_pixels_batch_filtered", n, data, len, flags, niter, layout, scale_denom,
			boxes != NULL, filter, boxes, out_on_device, out, max_device_bytes, rc, results, orientation, mode, thumbnail,
			reducing_gap, filters, nfilters);
}

extern "C" int jpegqs_cuda_pixels_batch_reduced(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const int32_t *orientation, int mode, int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results, int thumbnail, double reducing_gap) {
	return pixels_entry(ctx, "jpegqs_cuda_pixels_batch_reduced", n, data, len, flags, niter, layout, scale_denom,
			boxes != NULL, filter, boxes, out_on_device, out, max_device_bytes, rc, results, orientation, mode, thumbnail,
			reducing_gap);
}

extern "C" int jpegqs_cuda_pixels_batch_mode(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const int32_t *orientation, int mode, int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results) {
	return pixels_entry(ctx, "jpegqs_cuda_pixels_batch_mode", n, data, len, flags, niter, layout, scale_denom,
			boxes != NULL, filter, boxes, out_on_device, out, max_device_bytes, rc, results, orientation, mode);
}

extern "C" int jpegqs_cuda_pixels_batch_oriented(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const int32_t *orientation, int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results) {
	return pixels_entry(ctx, "jpegqs_cuda_pixels_batch_oriented", n, data, len, flags, niter, layout, scale_denom,
			boxes != NULL, filter, boxes, out_on_device, out, max_device_bytes, rc, results, orientation);
}

extern "C" int jpegqs_cuda_pixels_batch_resized(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes, int out_on_device,
		uint8_t *const *out, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results) {
	return pixels_entry(ctx, "jpegqs_cuda_pixels_batch_resized", n, data, len, flags, niter, layout, scale_denom, 1, filter, boxes,
			out_on_device, out, max_device_bytes, rc, results);
}

static int pixels_jpeg_entry(jpegqs_cuda_ctx *ctx, const char *who, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len, const int32_t *orientation, int mode, int thumbnail = 0, double gap = 0.0,
		const jpegqs_cuda_image_filter *filters = NULL, int nfilters = 0) {
	char msg[200];
	if (!ctx) return JPEGQS_ERR_ARG;
	if (n < 0) { snprintf(msg, sizeof(msg), "%s: negative file count", who); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
	if (!n) return 0;
	if (!data || !len || !out || !out_len || !rc || !results || !params) {
		snprintf(msg, sizeof(msg), "%s: NULL argument", who); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (params->quality < 1 || params->quality > 100 || params->subsampling < 0 || params->subsampling > 2 ||
			(params->optimize & ~(JPEGQS_JPEG_PROGRESSIVE | 1)) != 0) {
		snprintf(msg, sizeof(msg), "%s: params: quality outside 1..100, subsampling outside 0..2 or optimize other than 0 / 1 (| JPEGQS_JPEG_PROGRESSIVE)", who);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	for (int i = 0; i < n; i++) if (!data[i]) {
		snprintf(msg, sizeof(msg), "%s: file %d: NULL data", who, i);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (scale_denom != 1 && scale_denom != 2 && scale_denom != 4 && scale_denom != 8) {
		snprintf(msg, sizeof(msg), "%s: scale_denom must be 1, 2, 4 or 8", who); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (boxes) {
		if (!qs_resize_filter_ok(filter)) {
			snprintf(msg, sizeof(msg), "%s: filter %d: expected LANCZOS (1), BILINEAR (2), BICUBIC (3), BOX (4) or HAMMING (5)", who, filter);
			qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
		}
		for (int i = 0; i < n; i++) if (boxes[i].width < 1 || boxes[i].width > 65535 || boxes[i].height < 1 || boxes[i].height > 65535) {
			snprintf(msg, sizeof(msg), "%s: file %d: output size %d x %d outside 1..65535", who, i, boxes[i].width, boxes[i].height);
			qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
		}
	}
	if (!orientation_ok(ctx, who, n, orientation) || !mode_ok(ctx, who, mode) ||
			!reduced_ok(ctx, who, n, boxes, scale_denom, thumbnail, gap) || !filters_ok(ctx, who, filters, nfilters))
		return JPEGQS_ERR_ARG;
	for (int i = 0; i < n; i++) { memset(&results[i], 0, sizeof(results[i])); results[i].reason = ""; rc[i] = 0; out[i] = NULL; out_len[i] = 0; }
	return pixels_batch(ctx, who, n, data, len, flags, niter, JPEGQS_RENDER_HWC, scale_denom, filter, boxes, orientation, mode, 0, NULL,
			max_device_bytes, rc, results, params, out, out_len, thumbnail, gap, filters, nfilters);
}

extern "C" int jpegqs_cuda_pixels_batch_jpeg_filtered(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len, const int32_t *orientation, int mode, int thumbnail, double reducing_gap,
		const jpegqs_cuda_image_filter *filters, int nfilters) {
	return pixels_jpeg_entry(ctx, "jpegqs_cuda_pixels_batch_jpeg_filtered", n, data, len, flags, niter, scale_denom, filter, boxes,
			params, max_device_bytes, rc, results, out, out_len, orientation, mode, thumbnail, reducing_gap, filters, nfilters);
}

extern "C" int jpegqs_cuda_pixels_batch_jpeg_reduced(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len, const int32_t *orientation, int mode, int thumbnail, double reducing_gap) {
	return pixels_jpeg_entry(ctx, "jpegqs_cuda_pixels_batch_jpeg_reduced", n, data, len, flags, niter, scale_denom, filter, boxes,
			params, max_device_bytes, rc, results, out, out_len, orientation, mode, thumbnail, reducing_gap);
}

extern "C" int jpegqs_cuda_pixels_batch_jpeg(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len) {
	return pixels_jpeg_entry(ctx, "jpegqs_cuda_pixels_batch_jpeg", n, data, len, flags, niter, scale_denom, filter, boxes, params,
			max_device_bytes, rc, results, out, out_len, NULL, JPEGQS_PIXELS_AS_FILE);
}

extern "C" int jpegqs_cuda_pixels_batch_jpeg_oriented(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len, const int32_t *orientation) {
	return pixels_jpeg_entry(ctx, "jpegqs_cuda_pixels_batch_jpeg_oriented", n, data, len, flags, niter, scale_denom, filter, boxes,
			params, max_device_bytes, rc, results, out, out_len, orientation, JPEGQS_PIXELS_AS_FILE);
}

extern "C" int jpegqs_cuda_pixels_batch_jpeg_mode(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int scale_denom, int filter, const jpegqs_cuda_resize_box *boxes,
		const jpegqs_cuda_jpeg_params *params, size_t max_device_bytes, int *rc, jpegqs_cuda_pixels_result *results,
		uint8_t **out, size_t *out_len, const int32_t *orientation, int mode) {
	return pixels_jpeg_entry(ctx, "jpegqs_cuda_pixels_batch_jpeg_mode", n, data, len, flags, niter, scale_denom, filter, boxes,
			params, max_device_bytes, rc, results, out, out_len, orientation, mode);
}

extern "C" int jpegqs_cuda_pixels_batch_scaled(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int scale_denom, int out_on_device, uint8_t *const *out, size_t max_device_bytes,
		int *rc, jpegqs_cuda_pixels_result *results) {
	return pixels_entry(ctx, "jpegqs_cuda_pixels_batch_scaled", n, data, len, flags, niter, layout, scale_denom, 0, 0, NULL,
			out_on_device, out, max_device_bytes, rc, results);
}

extern "C" int jpegqs_cuda_pixels_batch(jpegqs_cuda_ctx *ctx, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int layout, int out_on_device, uint8_t *const *out, size_t max_device_bytes, int *rc,
		jpegqs_cuda_pixels_result *results) {
	return pixels_entry(ctx, "jpegqs_cuda_pixels_batch", n, data, len, flags, niter, layout, 1, 0, 0, NULL, out_on_device, out,
			max_device_bytes, rc, results);
}
