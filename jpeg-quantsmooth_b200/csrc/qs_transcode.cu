/*
 * qs_transcode.cu - jpegqs_cuda_transcode_batch and jpegqs_cuda_transcode (include/jpegqs_cuda.h):
 * JPEG files in host memory to the smoothed files the jpegqs tool writes, through the device
 * decoders, run_async and the device encoder on the context's stream, many files per launch.  The
 * decode, smoothing and encode kernels are those of qs_decode.cu, qs_scans.cu, qs_kernels.cu and
 * qs_encode.cu, reached through their public entry points; the one kernel here packs the encoded
 * files into one buffer so that a sub-batch comes back in one copy.
 */
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
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
	                                              packed files; the output slots */
	QsBuf stat_dev;                            /* per-file status words and the records of the packing kernel */
	QsBuf in_host, out_host, stat_host;        /* pinned staging of the upload and the two downloads */
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
	if (t->in_host.p) cudaFreeHost(t->in_host.p);
	if (t->out_host.p) cudaFreeHost(t->out_host.p);
	if (t->stat_host.p) cudaFreeHost(t->stat_host.p);
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

/* One file as the markers-only walk planned it, and what it needs of each buffer. */
struct QsPlan {
	jpegqs_cuda_image img; jpegqs_cuda_scan scan; jpegqs_cuda_jpeg_head head;
	std::vector<jpegqs_cuda_scan_rec> recs;    /* empty: one sequential scan (decode_async) */
	uint8_t *prefix; size_t plen;
	int smooth, can_up;
	size_t in_bytes, coef_bytes, up_bytes, cap;
	size_t ws_dec, ws_run, ws_enc;             /* this file's share of each stage's workspace */
};

/* bytes a sub-batch of these files needs: file + prefix + descriptor, coefficients (+ up-sampled
 * chroma), output slot, and the shared workspace - the largest of the three stages' and of the packed
 * output's.  Each stage's workspace formula is a sum over files (run_async's constant is counted per
 * file here, so this bounds the exact group figure from above). */
struct QsNeed {
	size_t fixed, dec, run, enc, packed;
	size_t total() const { size_t w = dec; if (run > w) w = run; if (enc > w) w = enc; if (packed > w) w = packed; return fixed + w; }
	void add(const QsPlan &p) {
		fixed += p.in_bytes + sizeof(QsPackDesc) + p.coef_bytes + p.up_bytes + align256(p.cap);
		dec += p.ws_dec; run += p.ws_run; enc += p.ws_enc; packed += align16(p.cap);
	}
};

/* the batch; `who` names the entry point in error messages */
static int transcode_batch(jpegqs_cuda_ctx *ctx, const char *who, int n, const uint8_t *const *data, const size_t *len,
		int flags, int niter, int optimize, int copy, size_t max_device_bytes, int *rc, jpegqs_cuda_transcode_result *results) {
	char msg[512];
	int device, sub_bytes; cudaStream_t st;
	std::vector<QsPlan> plans((size_t)n);
	for (int i = 0; i < n; i++) plans[i].prefix = NULL;
	int ret = 0;
#define TK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	snprintf(msg, sizeof(msg), "%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
	qs_ctx_decode_done(ctx, 0, msg); ret = JPEGQS_ERR_CUDA; goto fail; } } while (0)
#define TQ(call) do { int r_ = (call); if (r_ < 0) { ret = r_; goto fail; } } while (0)
	{
	qs_ctx_decode_info(ctx, &device, &st, &sub_bytes);
	QsTranscode **slot = (QsTranscode**)qs_ctx_transcode_state(ctx);
	TK(cudaSetDevice(device));
	if (!*slot) {
		QsTranscode *t = new QsTranscode();
		memset(t, 0, sizeof(*t));
		*slot = t;
		TK(cudaEventCreate(&t->ev0)); TK(cudaEventCreate(&t->ev1));
		TK(cudaDeviceGetAttribute(&t->sms, cudaDevAttrMultiProcessorCount, device));
	}
	QsTranscode *t = *slot;
	const int rflags = flags & QS_FLAGS_MASK;

	/* every file's route, and everything the stages need of it, from one markers-only walk */
	for (int i = 0; i < n; i++) {
		QsPlan &p = plans[i];
		int nscans = 0; const char *why;
		memset(&p.head, 0, sizeof(p.head));
		int route = qs_route_plan(data[i], len[i], copy, NULL, &p.img, &p.scan, t->recs, &nscans, &p.head, &p.prefix, &p.plen, &why);
		if (route < 0) {
			if (n == 1) snprintf(msg, sizeof(msg), "%s: %s", who, why);
			else snprintf(msg, sizeof(msg), "%s: file %d: %s", who, i, why);
			qs_ctx_decode_done(ctx, 0, msg);
			rc[i] = JPEGQS_ERR_ARG; continue;
		}
		if (route != JPEGQS_ROUTE_DEVICE) { results[i].reason = why; rc[i] = JPEGQS_TRANSCODE_FALLBACK; continue; }
		rc[i] = JPEGQS_TRANSCODE_OK;
		p.recs.assign(t->recs, t->recs + nscans);

		/* do_quantsmooth's early return (csrc/do_quantsmooth.c): nothing to smooth and nothing to
		 * up-sample leaves the coefficients and the quant tables as read */
		const jpegqs_cuda_comp *c = p.img.comp;
		int need_downsample = (flags & (QS_JOINT_YUV | QS_UPSAMPLE_UV)) && p.img.is_ycbcr && p.img.ncomp >= 3 &&
				c[1].h_samp == 1 && c[1].v_samp == 1 && c[2].h_samp == 1 && c[2].v_samp == 1;
		p.smooth = !((niter > QS_ITER_MAX ? QS_ITER_MAX : niter) <= 0 && !((flags & QS_UPSAMPLE_UV) && need_downsample));
		p.can_up = p.smooth && need_downsample && (flags & QS_UPSAMPLE_UV) && (c[0].h_samp != 1 || c[0].v_samp != 1);
		p.in_bytes = align256(len[i]) + align256(p.plen);
		p.coef_bytes = 0; p.up_bytes = 0;
		for (int k = 0; k < p.img.ncomp; k++) p.coef_bytes += align256((size_t)c[k].wblk * c[k].hblk * 128);
		if (p.can_up) p.up_bytes = 2 * align256((size_t)c[0].wblk * c[0].hblk * 128);
		if (p.recs.empty()) TQ(jpegqs_cuda_decode_workspace_bytes(1, &p.img, &p.scan, &len[i], &p.ws_dec));
		else {
			const jpegqs_cuda_scan_rec *r = p.recs.data();
			TQ(jpegqs_cuda_decode_scans_workspace_bytes(1, &p.img, &r, &nscans, &len[i], &p.ws_dec));
		}
		p.ws_run = 0;
		if (p.smooth) TQ(jpegqs_cuda_async_workspace_bytes(1, &p.img, rflags, &p.ws_run));
		TQ(jpegqs_cuda_encode_workspace_bytes(1, &p.img, optimize, &p.ws_enc));
		TQ(jpegqs_cuda_encode_bound(&p.img, p.plen, &p.cap));
	}

	/* the budget: 0 = half of what is free on the device now plus what these buffers already hold */
	size_t budget = max_device_bytes;
	if (!budget) {
		size_t fr = 0, tot = 0;
		TK(cudaMemGetInfo(&fr, &tot));
		budget = (fr + t->in_dev.cap + t->coef_dev.cap + t->ws_dev.cap + t->out_dev.cap + t->stat_dev.cap) / 2;
	}

	/* sub-batches: consecutive device files while their needs stay within the budget */
	int i0 = 0;
	while (i0 < n) {
		std::vector<int> files;
		QsNeed need = {0, 0, 0, 0, 0};
		int i = i0;
		for (; i < n && (int)files.size() < QS_PACK_MAX; i++) {
			if (rc[i] != JPEGQS_TRANSCODE_OK) continue;
			QsNeed with = need; with.add(plans[i]);
			if (!files.empty() && with.total() > budget) break;
			need = with; files.push_back(i);
		}
		i0 = i;
		if (files.empty()) continue;
		const int m = (int)files.size();

		/* encode order: the files that smooth first, so run_async's status array is a prefix of the
		 * encoder's; decoder statuses: the single-scan files, then the others */
		std::vector<int> order; order.reserve(m);
		for (int f : files) if (plans[f].smooth) order.push_back(f);
		const int ms = (int)order.size();
		for (int f : files) if (!plans[f].smooth) order.push_back(f);
		std::vector<jpegqs_cuda_image> eimg(m);
		std::vector<jpegqs_cuda_jpeg_head> heads(m);
		std::vector<uint8_t*> out_ptr(m);
		std::vector<size_t> caps(m);
		std::vector<QsPackDesc> desc(m);
		std::vector<int> seq_k, scan_k;                       /* encode positions of each decoder's files */
		for (int k = 0; k < m; k++) (plans[order[k]].recs.empty() ? seq_k : scan_k).push_back(k);

		/* exact workspace of each stage for this group; the packed output shares the workspace */
		size_t ws = 0, w, in_total = align256((size_t)m * sizeof(QsPackDesc)), coef_total = 0, out_total = 0, packed = 0;
		for (int k = 0; k < m; k++) eimg[k] = plans[order[k]].img;
		if (!seq_k.empty()) {
			std::vector<jpegqs_cuda_image> im; std::vector<jpegqs_cuda_scan> sc; std::vector<size_t> ln;
			for (int k : seq_k) { im.push_back(eimg[k]); sc.push_back(plans[order[k]].scan); ln.push_back(len[order[k]]); }
			TQ(jpegqs_cuda_decode_workspace_bytes((int)im.size(), im.data(), sc.data(), ln.data(), &w)); if (w > ws) ws = w;
		}
		if (!scan_k.empty()) {
			std::vector<jpegqs_cuda_image> im; std::vector<const jpegqs_cuda_scan_rec*> sc; std::vector<int> ns; std::vector<size_t> ln;
			for (int k : scan_k) {
				const QsPlan &p = plans[order[k]];
				im.push_back(eimg[k]); sc.push_back(p.recs.data()); ns.push_back((int)p.recs.size()); ln.push_back(len[order[k]]);
			}
			TQ(jpegqs_cuda_decode_scans_workspace_bytes((int)im.size(), im.data(), sc.data(), ns.data(), ln.data(), &w)); if (w > ws) ws = w;
		}
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
		std::vector<const uint8_t*> data_dev(m);
		for (int k = 0; k < m; k++) {
			QsPlan &p = plans[order[k]]; const size_t L = len[order[k]];
			jpegqs_cuda_image &im = eimg[k]; const jpegqs_cuda_comp *c = im.comp;
			for (int q = 0; q < im.ncomp; q++) { im.comp[q].coef = (int16_t*)cp; cp += align256((size_t)c[q].wblk * c[q].hblk * 128); }
			if (p.can_up) for (int q = 1; q <= 2; q++) { im.comp[q].coef_up = (int16_t*)cp; cp += p.up_bytes / 2; }
			memcpy(in_host + io, data[order[k]], L);
			memcpy(in_host + io + align256(L), p.prefix, p.plen);
			data_dev[k] = in_dev + io;
			heads[k] = p.head; heads[k].prefix_dev = in_dev + io + align256(L); heads[k].prefix_len = (uint32_t)p.plen;
			io += p.in_bytes;
			out_ptr[k] = (uint8_t*)t->out_dev.p + oo; caps[k] = p.cap;
			memset(&desc[k], 0, sizeof(desc[k]));
			desc[k].slot = oo; desc[k].cap = p.cap;
			oo += align256(p.cap);
		}
		for (size_t q = 0; q < seq_k.size(); q++) desc[seq_k[q]].dec_idx = (int32_t)q;
		for (size_t q = 0; q < scan_k.size(); q++) desc[scan_k[q]].dec_idx = (int32_t)(seq_k.size() + q);
		memcpy(in_host, desc.data(), (size_t)m * sizeof(QsPackDesc));
		TK(cudaMemcpyAsync(in_dev, in_host, in_total, cudaMemcpyHostToDevice, st));

		int32_t *dec = (int32_t*)(sd + st_dec), *enc = (int32_t*)(sd + st_enc);
		jpegqs_cuda_status *run = (jpegqs_cuda_status*)(sd + st_run);
		uint64_t *lens = (uint64_t*)(sd + st_len);
		if (!seq_k.empty()) {
			std::vector<jpegqs_cuda_image> im; std::vector<jpegqs_cuda_scan> sc; std::vector<const uint8_t*> dd; std::vector<size_t> ln;
			for (int k : seq_k) { im.push_back(eimg[k]); sc.push_back(plans[order[k]].scan); dd.push_back(data_dev[k]); ln.push_back(len[order[k]]); }
			TQ(jpegqs_cuda_decode_async(ctx, (int)im.size(), im.data(), sc.data(), dd.data(), ln.data(), t->ws_dev.p, t->ws_dev.cap, dec, st));
		}
		if (!scan_k.empty()) {
			std::vector<jpegqs_cuda_image> im; std::vector<const jpegqs_cuda_scan_rec*> sc; std::vector<int> ns;
			std::vector<const uint8_t*> dd; std::vector<size_t> ln;
			for (int k : scan_k) {
				const QsPlan &p = plans[order[k]];
				im.push_back(eimg[k]); sc.push_back(p.recs.data()); ns.push_back((int)p.recs.size());
				dd.push_back(data_dev[k]); ln.push_back(len[order[k]]);
			}
			TQ(jpegqs_cuda_decode_scans_async(ctx, (int)im.size(), im.data(), sc.data(), ns.data(), dd.data(), ln.data(),
					t->ws_dev.p, t->ws_dev.cap, dec + seq_k.size(), st));
		}
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
#undef TK
#undef TQ
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
