/*
 * qs_decode.h - the pieces of the device JPEG decoders that both qs_decode.cu (sequential files,
 * jpegqs_cuda_decode_async) and qs_scans.cu (any scan script, jpegqs_cuda_decode_scans_async) use:
 * the records in the workspace, the derived Huffman tables, the bit reader, the sequential unit
 * decoder, the subsequence spans and the byte passes (unstuffing, restart markers).
 */
#ifndef QS_DECODE_H
#define QS_DECODE_H
#include <cuda_runtime.h>
#include <cub/block/block_scan.cuh>
#include <cub/block/block_reduce.cuh>
#include <stdint.h>
#include <string.h>
#include "../../include/jpegqs_cuda.h"

#define HD __host__ __device__
#define QD_CHUNK 4096                  /* raw bytes per block of the byte passes             */
#define QD_BT 256                      /* threads of the byte passes: 16 bytes each          */
#define QD_ST 128                      /* subsequences per thread block of qd_sync / qd_final */
#define QD_SCAN_T 1024                 /* threads of the per-image scans                     */
#define QD_SUB_MIN 32
#define QD_SUB_DEFAULT 512
#define QD_MAX_UNITS 10                /* blocks per MCU (libjpeg D_MAX_BLOCKS_IN_MCU)        */
#define QD_PACK 8                      /* images per group (one setup launch)                */
#define QD_NONE (~0ull)
#define QD_FIXED 16384                 /* descriptor + state + 8 derived tables per image   */

/* zig-zag -> natural order (T.81 figure A.6) */
static __constant__ uint8_t qd_nat_dev[64] = {
	0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
	28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
	54, 47, 55, 62, 63 };
static const uint8_t qd_nat_host[64] = {
	0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
	28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
	54, 47, 55, 62, 63 };
HD static inline int qd_nat(int k) {
#ifdef __CUDA_ARCH__
	return qd_nat_dev[k];
#else
	return qd_nat_host[k];
#endif
}

/* ---------------------------------------------------------------- records */
struct QdHuff {                        /* derived decoding table of one DHT table */
	uint16_t look[512];                /* 9-bit prefix -> (length << 8) | symbol, 0 = longer code */
	int32_t maxcode[18];               /* largest code of each length, -1 = none             */
	int32_t valoff[17];                /* HUFFVAL index of code c of length l = valoff[l] + c */
	uint8_t val[256];
	uint32_t pad;
};
static_assert(sizeof(QdHuff) == 1424, "QdHuff");

struct QdImg {                         /* per-image descriptor (host-made, copied by qd_setup) */
	const uint8_t *data;               /* the file                                            */
	uint64_t off, len;                 /* entropy offset, file length                         */
	int16_t *coef[4];                  /* frame component arrays                              */
	uint32_t wblk[4], hblk[4];
	uint32_t nx, ny, nmcu;             /* MCUs per row / column (blocks for one component)    */
	uint32_t nblk, period, ri, nint_cap;
	uint32_t nchunk, sub_bytes, nsub_cap, pad0;
	uint8_t u_comp[QD_MAX_UNITS], u_h[QD_MAX_UNITS], u_v[QD_MAX_UNITS], u_hs[QD_MAX_UNITS], u_vs[QD_MAX_UNITS];
	uint8_t u_dc[QD_MAX_UNITS], u_ac[QD_MAX_UNITS];        /* table slots of unit k of the MCU */
	uint8_t pad1[2];
	/* workspace */
	QdHuff *tab;                       /* [8]: DC 0..3, AC 0..3                                */
	struct QdState *st;
	uint8_t *unst;                     /* the segment without FF00 stuffing and RST markers    */
	struct QdChunk *chunk;
	uint32_t *ivstart, *ivsub0;        /* per restart interval: first byte, first subsequence */
	struct QdSub *sub;
	int32_t *status;
};

struct QdState {                       /* per image, written on the device */
	uint32_t nbytes, nrst, nint, nsub, termchunk, pad[3];
};
struct QdChunk { uint32_t kept, rst, term, kbase, rbase, pad; };
struct QdSub {
	uint64_t entry, exit;              /* (bit position << 4) | phase; entry QD_NONE = not decoded */
	uint64_t err;                      /* (unit start << 8) | JPEGQS_DECODE_* bits of the path's last error */
	uint32_t cnt, iv;                  /* units from entry to exit; restart interval          */
	int32_t dcs[QD_MAX_UNITS];         /* DC differences summed per unit index mod nblk       */
	uint32_t g0, sync_units;           /* first unit inside the interval; units re-decoded    */
	int32_t pred[4];                   /* DC predictors at entry, per scan component          */
};
static_assert(sizeof(QdSub) == 96, "jpegqs_cuda.h: 96 bytes per subsequence");
static_assert(sizeof(QdChunk) == 24, "jpegqs_cuda.h: 24 bytes per chunk");
static_assert(sizeof(QdImg) <= 1024 && sizeof(QdState) <= 1024 && 2048 + 8 * sizeof(QdHuff) <= QD_FIXED, "fixed part");

/* ---------------------------------------------------------------- table building (host + device) */
HD static inline int qd_build(QdHuff *h, const uint8_t *bits, const uint8_t *val) {
	int code = 0, k = 0;
	for (int i = 0; i < 512; i++) h->look[i] = 0;
	for (int l = 1; l <= 16; l++) {
		h->valoff[l] = k - code;
		for (int i = 0; i < bits[l]; i++, k++, code++) {
			if (k >= 256 || code >= (1 << l)) return -1;
			if (l <= 9) for (int j = 0; j < (1 << (9 - l)); j++) h->look[(code << (9 - l)) + j] = (uint16_t)((l << 8) | val[k]);
		}
		h->maxcode[l] = bits[l] ? code - 1 : -1;
		if (code >= (1 << l) && bits[l]) return -1;
		code <<= 1;
	}
	h->maxcode[17] = 0x7fffffff; h->maxcode[0] = -1; h->valoff[0] = 0;
	for (int i = 0; i < 256; i++) h->val[i] = val[i];
	h->pad = 0;
	return 0;
}

/* ---------------------------------------------------------------- the bit reader and the unit decoder */
struct QdRd { const uint8_t *d; uint32_t lim; };        /* bytes at or past lim read as 0 */

HD static inline uint32_t qd_peek32(const QdRd &r, uint64_t pos) {
	uint64_t b = pos >> 3, w = 0;
	for (int i = 0; i < 5; i++) w = (w << 8) | (b + i < r.lim ? r.d[b + i] : 0u);
	return (uint32_t)(w >> (8 - (pos & 7)));
}
HD static inline int qd_sym(const QdHuff *h, uint32_t w, int *len) {
	uint32_t e = h->look[w >> 23];
	if (e) { *len = (int)(e >> 8); return (int)(e & 255); }
	for (int l = 10; l <= 16; l++) {
		int code = (int)(w >> (32 - l));
		if (code <= h->maxcode[l]) { *len = l; return h->val[h->valoff[l] + code]; }
	}
	*len = 0;
	return 0;
}
HD static inline int qd_extend(uint32_t v, int s) { return s && v < (1u << (s - 1)) ? (int)v + 1 - (1 << s) : (int)v; }

/* one unit at bit position pos; returns the position after it.  blk (may be NULL): natural-order
 * coefficients, written where non-zero (the caller clears it).  A bad code consumes 16 bits and reads
 * as symbol 0, as jpegcoef.c does, so every decode is deterministic and bounded. */
HD static inline uint64_t qd_unit(const QdRd &r, uint64_t pos, const QdHuff *dc, const QdHuff *ac, int *diff,
		int16_t *blk, uint32_t *err) {
	int len, s;
	uint32_t w = qd_peek32(r, pos);
	s = qd_sym(dc, w, &len);
	if (!len) { *err |= JPEGQS_DECODE_BAD_CODE; len = 16; s = 0; }
	s &= 15;
	*diff = s ? qd_extend((w << len) >> (32 - s), s) : 0;
	pos += (uint64_t)(len + s);
	for (int k = 1; k < 64; ) {
		w = qd_peek32(r, pos);
		int rs = qd_sym(ac, w, &len);
		if (!len) { *err |= JPEGQS_DECODE_BAD_CODE; len = 16; rs = 0; }
		int run = rs >> 4; s = rs & 15;
		if (s) {
			k += run;
			if (k > 63) *err |= JPEGQS_DECODE_AC_RUN;
			else if (blk) blk[qd_nat(k)] = (int16_t)qd_extend((w << len) >> (32 - s), s);
			pos += (uint64_t)(len + s);
			k++;
		} else {
			pos += (uint64_t)len;
			if (run != 15) break;
			k += 16;
		}
	}
	if (pos > 8ull * r.lim) *err |= JPEGQS_DECODE_TRUNCATED;
	return pos;
}

/* the remaining bits up to the interval end are padding: fewer than 8, all ones (F.1.2.3) */
HD static inline bool qd_padding(const QdRd &r, uint64_t a, uint64_t iv_end) {
	if (a >= iv_end) return true;
	uint64_t nb = iv_end - a;
	if (nb >= 8) return false;
	uint32_t w = qd_peek32(r, a) >> (32 - nb);
	return w == (1u << nb) - 1;
}

/* subsequence s of an image: its interval, bit range, whether it is the interval's last */
struct QdSpan { uint32_t iv; uint64_t begin, end, iv_end; bool first, last; };
HD static inline QdSpan qd_span(const QdImg &im, const uint32_t *ivstart, const uint32_t *ivsub0, uint32_t nint,
		uint32_t nbytes, uint32_t nsub, uint32_t s) {
	uint32_t lo = 0, hi = nint - 1;                     /* last interval with ivsub0 <= s */
	while (lo < hi) { uint32_t mid = (lo + hi + 1) >> 1; if (ivsub0[mid] <= s) lo = mid; else hi = mid - 1; }
	QdSpan sp;
	sp.iv = lo;
	uint32_t b0 = ivstart[lo], b1 = lo + 1 < nint ? ivstart[lo + 1] : nbytes;
	uint32_t j = s - ivsub0[lo], nsj = lo + 1 < nint ? ivsub0[lo + 1] - ivsub0[lo] : nsub - ivsub0[lo];
	uint64_t x0 = (uint64_t)b0 + (uint64_t)j * im.sub_bytes, x1 = x0 + im.sub_bytes;
	if (x1 > b1 || j + 1 == nsj) x1 = b1;
	if (x0 > b1) x0 = b1;
	sp.begin = 8 * x0; sp.end = 8 * x1; sp.iv_end = 8ull * b1;
	sp.first = j == 0; sp.last = j + 1 == nsj;
	return sp;
}

/* units expected in interval k */
HD static inline int64_t qd_expect(const QdImg &im, uint32_t k, uint32_t nint) {
	if (!im.ri) return (int64_t)im.nmcu * im.nblk;
	int64_t m = k + 1 < nint ? (int64_t)im.ri : (int64_t)im.nmcu - (int64_t)(nint - 1) * im.ri;
	return (m < 0 ? 0 : m) * im.nblk;
}

/* ---------------------------------------------------------------- byte passes: rules shared by host and device
 * Position p of [off, len) is a terminator when data[p] = FF and the next byte is neither 00 nor
 * (with restarts) RSTn, or there is none; it is kept (part of the unstuffed data) when it lies
 * before the first terminator, does not follow an FF, and is not the FF of an RSTn; it starts an
 * RSTn when data[p] = FF is followed by D0..D7 (restarts only). */
HD static inline void qd_byte_class(const uint8_t *d, uint64_t off, uint64_t len, uint64_t p, bool ri,
		bool *term, bool *keep, bool *rst) {
	uint8_t x = d[p];
	uint8_t nx = p + 1 < len ? d[p + 1] : 0;
	bool last = p + 1 >= len;
	bool isrst = x == 0xFF && !last && (nx & 0xF8) == 0xD0;
	*term = x == 0xFF && (last || (nx != 0 && !(ri && isrst)));
	*rst = ri && isrst;
	*keep = !(p > off && d[p - 1] == 0xFF) && !(x == 0xFF && isrst);
}

/* per chunk c of QD_CHUNK raw bytes: the first terminator, kept bytes and RSTn before it (QD_BT threads) */
static __device__ __forceinline__ void qd_scan_body(const QdImg &im, uint32_t c) {
	if (c >= im.nchunk) return;
	typedef cub::BlockReduce<uint32_t, QD_BT> R;
	__shared__ typename R::TempStorage tmp;
	__shared__ uint32_t s_term;
	uint64_t p0 = im.off + (uint64_t)c * QD_CHUNK + threadIdx.x * 16;
	uint32_t term = 0xFFFFFFFFu;
	bool ri = im.ri != 0;
	for (int j = 0; j < 16; j++) {
		uint64_t p = p0 + j;
		if (p >= im.len) break;
		bool t, k, r;
		qd_byte_class(im.data, im.off, im.len, p, ri, &t, &k, &r);
		if (t) { term = (uint32_t)(p - im.off); break; }
	}
	uint32_t bt = R(tmp).Reduce(term, cub::Min());
	if (threadIdx.x == 0) s_term = bt;
	__syncthreads();
	bt = s_term;
	uint32_t kept = 0, rst = 0;
	for (int j = 0; j < 16; j++) {
		uint64_t p = p0 + j;
		if (p >= im.len || p - im.off >= bt) break;
		bool t, k, r;
		qd_byte_class(im.data, im.off, im.len, p, ri, &t, &k, &r);
		kept += k; rst += r;
	}
	__syncthreads();
	uint32_t sk = R(tmp).Sum(kept);
	__syncthreads();
	uint32_t sr = R(tmp).Sum(rst);
	if (threadIdx.x == 0) { QdChunk &ch = im.chunk[c]; ch.kept = sk; ch.rst = sr; ch.term = bt; }
}

/* per image: prefix of the chunk counts up to the first terminator; segment length, RSTn count (QD_SCAN_T threads) */
static __device__ __forceinline__ void qd_seg_body(const QdImg &im) {
	typedef cub::BlockScan<uint2, QD_SCAN_T> S;
	typedef cub::BlockReduce<uint32_t, QD_SCAN_T> R;
	__shared__ union { typename S::TempStorage s; typename R::TempStorage r; } tmp;
	__shared__ uint32_t s_stop;
	uint2 carry = make_uint2(0, 0);
	uint32_t stop = im.nchunk;
	for (uint32_t base = 0; base < im.nchunk && base < stop; base += QD_SCAN_T) {
		uint32_t c = base + threadIdx.x;
		uint2 v = make_uint2(0, 0); uint32_t t = 0xFFFFFFFFu;
		if (c < im.nchunk) { QdChunk ch = im.chunk[c]; v = make_uint2(ch.kept, ch.rst); if (ch.term != 0xFFFFFFFFu) t = c; }
		uint32_t first = R(tmp.r).Reduce(t, cub::Min());
		if (threadIdx.x == 0) s_stop = first;
		__syncthreads();
		first = s_stop;
		if (c > first) v = make_uint2(0, 0);
		uint2 ex, agg;
		struct Add { __device__ uint2 operator()(uint2 a, uint2 b) const { return make_uint2(a.x + b.x, a.y + b.y); } };
		S(tmp.s).ExclusiveScan(v, ex, make_uint2(0, 0), Add(), agg);
		if (c < im.nchunk && c <= first) { im.chunk[c].kbase = carry.x + ex.x; im.chunk[c].rbase = carry.y + ex.y; }
		carry.x += agg.x; carry.y += agg.y;
		if (first != 0xFFFFFFFFu) stop = first;
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		QdState *st = im.st;
		st->nbytes = carry.x; st->nrst = carry.y; st->termchunk = stop;
		uint32_t nint = im.ri ? carry.y + 1 : 1;
		if (im.ri && nint != im.nint_cap) atomicOr(im.status, JPEGQS_DECODE_RESTART);
		if (nint > im.nint_cap) nint = im.nint_cap;
		st->nint = nint;
		im.ivstart[0] = 0;
	}
}

/* per chunk c: writes the kept bytes and the restart positions, checks the RSTn sequence (QD_BT threads) */
static __device__ __forceinline__ void qd_compact_body(const QdImg &im, uint32_t c) {
	if (c >= im.nchunk || c > im.st->termchunk) return;
	QdChunk ch = im.chunk[c];
	typedef cub::BlockScan<uint32_t, QD_BT> S;
	__shared__ typename S::TempStorage tmp;
	uint64_t p0 = im.off + (uint64_t)c * QD_CHUNK + threadIdx.x * 16;
	bool ri = im.ri != 0;
	uint32_t mk = 0, mr = 0, nk = 0, nr = 0;
	for (int j = 0; j < 16; j++) {
		uint64_t p = p0 + j;
		if (p >= im.len || p - im.off >= ch.term) break;
		bool t, k, r;
		qd_byte_class(im.data, im.off, im.len, p, ri, &t, &k, &r);
		mk |= (uint32_t)k << j; mr |= (uint32_t)r << j; nk += k; nr += r;
	}
	uint32_t packed = nk | nr << 16, ex;
	S(tmp).ExclusiveSum(packed, ex);
	uint32_t ko = ch.kbase + (ex & 0xFFFF), ro = ch.rbase + (ex >> 16);
	uint32_t nint = im.st->nint;
	for (int j = 0; j < 16; j++) {
		uint64_t p = p0 + j;
		if (mr >> j & 1) {
			if ((uint32_t)(im.data[p + 1] & 7) != (ro & 7)) atomicOr(im.status, JPEGQS_DECODE_RESTART);
			if (ro + 1 < nint) im.ivstart[ro + 1] = ko;
			ro++;
		}
		if (mk >> j & 1) im.unst[ko++] = im.data[p];
	}
}

/* per image: subsequences per interval and their prefix (QD_SCAN_T threads) */
static __device__ __forceinline__ void qd_iv_body(const QdImg &im) {
	QdState *st = im.st;
	typedef cub::BlockScan<uint32_t, QD_SCAN_T> S;
	__shared__ typename S::TempStorage tmp;
	uint32_t nint = st->nint, nbytes = st->nbytes, carry = 0;
	for (uint32_t base = 0; base < nint; base += QD_SCAN_T) {
		uint32_t k = base + threadIdx.x, ns = 0;
		if (k < nint) {
			uint32_t b0 = im.ivstart[k], b1 = k + 1 < nint ? im.ivstart[k + 1] : nbytes;
			if (b1 < b0) { b1 = b0; atomicOr(im.status, JPEGQS_DECODE_RESTART); }
			ns = (b1 - b0 + im.sub_bytes - 1) / im.sub_bytes;
			if (!ns) ns = 1;
		}
		uint32_t ex, agg;
		S(tmp).ExclusiveSum(ns, ex, agg);
		if (k < nint) im.ivsub0[k] = carry + ex;
		carry += agg;
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		if (carry > im.nsub_cap) { carry = im.nsub_cap; atomicOr(im.status, JPEGQS_DECODE_UNITS); }
		st->nsub = carry;
	}
}

#endif
