/*
 * qs_scans.cu - jpegqs_cuda_decode_scans_async: JPEG files of any scan script (progressive, several
 * sequential scans) decoded to quantized coefficients on the GPU, and jpegqs_cuda_decode_scans_model,
 * the same steps on the CPU.  DESIGN.md section 3.6.1 describes the scheme; in short, every scan is
 * a segment of its own, run through decode_async's machinery (qs_decode.h) where that applies:
 *
 *   kind       SEQ  a sequential scan (interleaved or not): decode_async's unit.
 *              DCF  a progressive DC first scan: the DC code and its bits; values stored << Al.
 *              ACF  a progressive AC first scan (one component): one block's band, or an end-of-band
 *                   run, which is one decoder STEP that counts all the blocks of the run.  The state
 *                   at a step boundary is the bit position alone (period 1).
 *              DCR  a DC refinement scan: bit j of a restart interval is its block j.
 *              ACR  an AC refinement scan: reads each block's coefficients as they stand.
 *   bytes      one unstuff / RSTn pass over every scan of every image (qd_scan / qd_seg / qd_compact).
 *   first      SEQ, DCF and ACF scans: speculative subsequences, synchronisation, chain, placement
 *              and final decode, all scans of a group in one set of launches.  A run that outlives
 *              its restart interval or scan is cut there, as libjpeg does.
 *   DCR        one launch for every DC refinement scan: blk[0] |= 1 << Al commutes across scans.
 *   ACR        one launch per level; one thread decodes one restart interval serially, with the
 *              already non-zero coefficients from a 64-bit mask (skip by __fns, count by __popcll).
 */
#include <stdio.h>
#include <memory>
#include <vector>
#include <algorithm>
#include "qs_decode.h"

enum { QS_SEQ = 0, QS_DCF = 1, QS_ACF = 2, QS_DCR = 3, QS_ACR = 4 };
#define QS_GROUP_IMGS 16               /* images per group                                    */
#define QS_GROUP_SEGS 512              /* scans per group                                     */
#define QS_PACK 24                     /* scans per store launch                              */
#define QS_PACK_TABS 48                /* Huffman tables per store launch                     */
#define QS_RT 128                      /* threads of the AC refinement kernel: 4 intervals    */

struct QsSeg {                         /* per scan, at the start of its workspace */
	QdImg im;                          /* the scan as decode_async sees an image: nx / ny / units / tables */
	uint32_t kind, Ss, Se, Al, level, pad[3];
};
static_assert(sizeof(QsSeg) <= 1024, "descriptor");

/* ---------------------------------------------------------------- steps: one decoder step from a state */
struct QsView {
	const QdHuff *dc[QD_MAX_UNITS], *ac[QD_MAX_UNITS];   /* by phase */
	uint32_t period, nblk, kind, Ss, Se, Al;
	QdRd rd;
};
HD static inline void qs_view(const QsSeg &s, const QdHuff *tab, const uint8_t *unst, uint32_t lim, QsView *v) {
	const QdImg &im = s.im;
	for (uint32_t p = 0; p < im.period; p++) { v->dc[p] = tab + im.u_dc[p]; v->ac[p] = tab + 4 + im.u_ac[p]; }
	v->period = im.period; v->nblk = im.nblk; v->rd.d = unst; v->rd.lim = lim;
	v->kind = s.kind; v->Ss = s.Ss; v->Se = s.Se; v->Al = s.Al;
}

/* one step at bit position pos, phase ph: *units blocks (1, or an ACF end-of-band run), *diff the DC
 * difference.  blk (may be NULL): SEQ a cleared natural-order block to fill; ACF the destination block
 * (coded coefficients written << Al); unused otherwise. */
HD static inline uint64_t qs_step(const QsView &v, uint64_t pos, uint32_t ph, int *diff, uint32_t *units, int16_t *blk,
		uint32_t *err) {
	*units = 1; *diff = 0;
	if (v.kind == QS_SEQ) return qd_unit(v.rd, pos, v.dc[ph], v.ac[ph], diff, blk, err);
	int len, s;
	uint32_t w = qd_peek32(v.rd, pos);
	if (v.kind == QS_DCF) {
		s = qd_sym(v.dc[ph], w, &len);
		if (!len) { *err |= JPEGQS_DECODE_BAD_CODE; len = 16; s = 0; }
		s &= 15;
		*diff = s ? qd_extend((w << len) >> (32 - s), s) : 0;
		pos += (uint64_t)(len + s);
	} else {
		const QdHuff *h = v.ac[0];
		for (int k = (int)v.Ss; k <= (int)v.Se; ) {
			w = qd_peek32(v.rd, pos);
			int rs = qd_sym(h, w, &len);
			if (!len) { *err |= JPEGQS_DECODE_BAD_CODE; len = 16; rs = 0; }
			int r = rs >> 4; s = rs & 15;
			if (s) {
				k += r;
				if (k > (int)v.Se) *err |= JPEGQS_DECODE_AC_RUN;
				else if (blk) blk[qd_nat(k)] = (int16_t)(qd_extend((w << len) >> (32 - s), s) * (1 << v.Al));
				pos += (uint64_t)(len + s);
				k++;
			} else if (r == 15) {
				pos += (uint64_t)len;
				k += 16;
			} else {                                    /* EOBr: this block and (2^r - 1 + bits) more */
				*units = (1u << r) + (r ? (w << len) >> (32 - r) : 0u);
				pos += (uint64_t)(len + r);
				break;
			}
		}
	}
	if (pos > 8ull * v.rd.lim) *err |= JPEGQS_DECODE_TRUNCATED;
	return pos;
}

/* qd_path with steps: decodes from state `start` until a step start at or past end_bits (or the
 * padding before the interval end when last); with old, runs beside that decode and stops where the
 * two meet.  Counts are units (blocks). */
HD static uint32_t qs_path(const QsView &v, uint64_t start, uint64_t end_bits, uint64_t iv_end, bool last,
		const QdSub *old, QdSub *out) {
	uint64_t a = start >> 4, b = 0; uint32_t pa = (uint32_t)(start & 15), pb = 0, ca = 0, cb = 0, ra = 0, rb = 0, n = 0;
	int32_t da[QD_MAX_UNITS], db[QD_MAX_UNITS];
	uint64_t ea = 0;
	bool hasb = old && old->entry != QD_NONE;
	for (int i = 0; i < QD_MAX_UNITS; i++) da[i] = db[i] = 0;
	if (hasb) { b = old->entry >> 4; pb = (uint32_t)(old->entry & 15); }
	for (;;) {
		if (hasb && a == b && pa == pb) {
			uint32_t sh = (ca + v.nblk - cb % v.nblk) % v.nblk;
			int32_t d[QD_MAX_UNITS];
			for (uint32_t r = 0; r < v.nblk; r++) d[r] = da[r];
			for (uint32_t r = 0; r < v.nblk; r++) d[(r + sh) % v.nblk] += old->dcs[r] - db[r];
			for (uint32_t r = 0; r < v.nblk; r++) out->dcs[r] = d[r];
			out->cnt = ca + (old->cnt - cb);
			out->exit = old->exit;
			out->err = old->err && (old->err >> 8) >= b ? old->err : ea;
			break;
		}
		bool end = a >= end_bits || (last && qd_padding(v.rd, a, iv_end));
		if (end) {
			for (uint32_t r = 0; r < v.nblk; r++) out->dcs[r] = da[r];
			out->cnt = ca; out->exit = a << 4 | pa; out->err = ea;
			break;
		}
		uint32_t e = 0, nu; int diff;
		if (!hasb || cb >= old->cnt || a <= b) {
			uint64_t na = qs_step(v, a, pa, &diff, &nu, NULL, &e);
			if (e) ea = a << 8 | e;
			da[ra] += diff; ra = ra + 1 == v.nblk ? 0 : ra + 1;
			a = na; pa = pa + 1 == v.period ? 0 : pa + 1; ca += nu; n += nu;
		} else {
			uint64_t nb = qs_step(v, b, pb, &diff, &nu, NULL, &e);
			db[rb] += diff; rb = rb + 1 == v.nblk ? 0 : rb + 1;
			b = nb; pb = pb + 1 == v.period ? 0 : pb + 1; cb += nu;
		}
	}
	out->entry = start;
	return n;
}

/* the final decode of a subsequence into the arrays (v: tables by unit index, period = nblk) */
HD static inline uint32_t qs_final_sub(const QsSeg &sg, const QsView &v, const QdSub &sb, uint32_t nint) {
	const QdImg &im = sg.im;
	uint32_t err = 0;
	if (sb.entry == QD_NONE) return 0;
	uint64_t pos = sb.entry >> 4;
	int32_t pred[4] = { sb.pred[0], sb.pred[1], sb.pred[2], sb.pred[3] };
	uint64_t base = (uint64_t)sb.iv * im.ri * im.nblk, lim = base + (uint64_t)qd_expect(im, sb.iv, nint);
	uint64_t u = base + sb.g0;
	for (uint32_t done = 0; done < sb.cnt; ) {
		uint32_t k = (uint32_t)(u % im.nblk), c = im.u_comp[k], nu; uint64_t m = u / im.nblk;
		int16_t *dst = NULL; int diff;
		if (m < im.nmcu) {
			uint64_t bx = (uint64_t)(m % im.nx) * im.u_hs[k] + im.u_h[k], by = (uint64_t)(m / im.nx) * im.u_vs[k] + im.u_v[k];
			if (bx < im.wblk[c] && by < im.hblk[c]) dst = im.coef[c] + ((size_t)by * im.wblk[c] + bx) * 64;
		} else if (sg.kind != QS_ACF) err |= JPEGQS_DECODE_UNITS;
		if (sg.kind == QS_SEQ) {
			int16_t blk[64];
			for (int j = 0; j < 64; j++) blk[j] = 0;
			pos = qs_step(v, pos, k, &diff, &nu, blk, &err);
			pred[c] += diff;
			blk[0] = (int16_t)pred[c];
			if (dst) {
#ifdef __CUDA_ARCH__
				for (int j = 0; j < 8; j++) reinterpret_cast<int4 *>(dst)[j] = reinterpret_cast<const int4 *>(blk)[j];
#else
				memcpy(dst, blk, sizeof(blk));
#endif
			}
		} else if (sg.kind == QS_DCF) {
			pos = qs_step(v, pos, k, &diff, &nu, NULL, &err);
			pred[c] += diff;
			if (dst) dst[0] = (int16_t)(pred[c] * (1 << sg.Al));
		} else pos = qs_step(v, pos, 0, &diff, &nu, u < lim ? dst : NULL, &err);
		done += nu; u += nu;
	}
	if (pos != sb.exit >> 4) err |= JPEGQS_DECODE_UNITS;
	return err;
}

/* ---------------------------------------------------------------- refinement scans */
/* which AC coefficients of a block are not zero, as a zig-zag mask: entry (r, b) of the table is the
 * zig-zag mask of row r's natural-order non-zero pattern b (host and device fill it with this) */
HD static inline uint64_t qs_zz_entry(int r, int b) {
	uint64_t m = 0;
	for (int k = 0; k < 64; k++) { int n = qd_nat(k); if (n >> 3 == r && (b >> (n & 7) & 1)) m |= 1ull << k; }
	return m;
}
HD static inline uint64_t qs_nzmask(const int16_t *blk, const uint64_t (*tab)[256]) {
	uint64_t m = 0;
	for (int r = 0; r < 8; r++) {
		uint32_t b = 0;
		for (int j = 0; j < 8; j++) b |= (uint32_t)(blk[r * 8 + j] != 0) << j;
		m |= tab[r][b];
	}
	return m & ~1ull;
}
#ifdef __CUDA_ARCH__
/* the same from the block's eight 16-byte rows in registers */
static __device__ __forceinline__ uint64_t qs_nzmask_rows(const int4 *q, const uint64_t (*tab)[256]) {
	uint64_t m = 0;
	for (int r = 0; r < 8; r++) {
		uint32_t x[4] = { (uint32_t)q[r].x, (uint32_t)q[r].y, (uint32_t)q[r].z, (uint32_t)q[r].w }, b = 0;
		for (int j = 0; j < 4; j++) b |= (uint32_t)((x[j] & 0xFFFF) != 0) << (2 * j) | (uint32_t)((x[j] >> 16) != 0) << (2 * j + 1);
		m |= tab[r][b];
	}
	return m & ~1ull;
}
#endif
/* the position of the n-th (0-based) set bit of m, 64 if there is none */
HD static inline int qs_nth(uint64_t m, int n) {
#ifdef __CUDA_ARCH__
	uint32_t lo = (uint32_t)m, c = __popc(lo);
	if ((uint32_t)n < c) return (int)__fns(lo, 0, n + 1);
	uint32_t r = __fns((uint32_t)(m >> 32), 0, n - (int)c + 1);
	return r == 0xFFFFFFFFu ? 64 : 32 + (int)r;
#else
	for (; n > 0 && m; n--) m &= m - 1;
	return m ? __builtin_ctzll(m) : 64;
#endif
}
HD static inline int qs_ctz(uint64_t m) {
#ifdef __CUDA_ARCH__
	return __ffsll((long long)m) - 1;
#else
	return __builtin_ctzll(m);
#endif
}

/* a bit window in registers over unstuffed bytes [p, lim); bytes past lim read as 0 */
struct QsBits {
	const uint8_t *d; uint32_t p, lim; int n; uint64_t buf, used;
	HD inline void fill() { while (n <= 56) { buf |= (uint64_t)(p < lim ? d[p] : 0u) << (56 - n); p++; n += 8; } }
	HD inline uint32_t peek32() { if (n < 32) fill(); return (uint32_t)(buf >> 32); }
	HD inline void skip(int k) { buf <<= k; n -= k; used += (uint64_t)k; }
	HD inline uint32_t get(int k) { if (!k) return 0; uint32_t v = peek32() >> (32 - k); skip(k); return v; }
};

/* one restart interval (the whole scan without restarts) of an AC refinement scan: blocks
 * [u0, u0 + nu) of the component, unstuffed bytes [b0, b1); G.1.2.3 as libjpeg decodes it */
HD static uint32_t qs_acr_interval(const QsSeg &sg, const QdHuff *ac, const uint8_t *unst, uint32_t b0, uint32_t b1,
		uint64_t u0, uint64_t nu, const uint64_t (*tab)[256]) {
	const QdImg &im = sg.im;
	int16_t *arr = im.coef[im.u_comp[0]];
	const int Ss = (int)sg.Ss, Se = (int)sg.Se, p1 = 1 << sg.Al, m1 = -p1;
	const uint64_t range = (Se == 63 ? ~0ull : (1ull << (Se + 1)) - 1) & (~0ull << Ss);
	QsBits br; br.d = unst; br.p = b0; br.lim = b1; br.n = 0; br.buf = 0; br.used = 0;
	uint32_t err = 0, eobrun = 0;
#ifdef __CUDA_ARCH__
	/* the next block's rows are loaded while this one decodes: the blocks of an interval are read in
	 * order, and a scan writes only the block it decodes */
	int4 nxt[8];
	if (nu) for (int r = 0; r < 8; r++) nxt[r] = reinterpret_cast<const int4 *>(arr + (size_t)u0 * 64)[r];
#endif
	for (uint64_t i = 0; i < nu; i++) {
		int16_t *blk = arr + (size_t)(u0 + i) * 64;       /* one component, not interleaved: block = unit */
#ifdef __CUDA_ARCH__
		int4 cur[8];
		for (int r = 0; r < 8; r++) cur[r] = nxt[r];
		if (i + 1 < nu) for (int r = 0; r < 8; r++) nxt[r] = reinterpret_cast<const int4 *>(blk + 64)[r];
		const uint64_t nz = qs_nzmask_rows(cur, tab) & range;
#else
		const uint64_t nz = qs_nzmask(blk, tab) & range;
#endif
		int k = Ss;
		if (!eobrun) {
			while (k <= Se) {
				int len, rs = qd_sym(ac, br.peek32(), &len);
				if (!len) { err |= JPEGQS_DECODE_BAD_CODE; len = 16; rs = 0; }
				br.skip(len);
				int r = rs >> 4, s = rs & 15, val = 0;
				if (s) val = br.get(1) ? p1 : m1;
				else if (r != 15) { eobrun = (1u << r) + br.get(r); break; }
				/* skip r zero-history coefficients; the non-zero ones passed take a correction bit */
				int t = qs_nth(~nz & range & (~0ull << k), r);
				if (t > Se) t = Se + 1;
				uint64_t w = nz & (~0ull << k) & (t > 63 ? ~0ull : (1ull << t) - 1);
				while (w) {
					int j = qs_ctz(w); w &= w - 1;
					if (br.get(1)) { int16_t *cp = blk + qd_nat(j); if (!(*cp & p1)) *cp = (int16_t)(*cp + (*cp >= 0 ? p1 : m1)); }
				}
				k = t;
				if (val) { if (k <= Se) blk[qd_nat(k)] = (int16_t)val; else err |= JPEGQS_DECODE_AC_RUN; }
				k++;
			}
		}
		if (eobrun) {
			if (k <= Se) {
				uint64_t w = nz & (~0ull << k);
				while (w) {
					int j = qs_ctz(w); w &= w - 1;
					if (br.get(1)) { int16_t *cp = blk + qd_nat(j); if (!(*cp & p1)) *cp = (int16_t)(*cp + (*cp >= 0 ? p1 : m1)); }
				}
			}
			eobrun--;
		}
	}
	if (br.used > 8ull * (b1 - b0)) err |= JPEGQS_DECODE_TRUNCATED;
	return err;
}

/* unit u of a DC refinement scan: its block (NULL outside the image), whether its bit is set */
HD static inline uint32_t qs_dcr_unit(const QsSeg &sg, const uint8_t *unst, const uint32_t *ivstart, uint32_t nint,
		uint32_t nbytes, uint64_t u, int16_t **dst, bool *one) {
	const QdImg &im = sg.im;
	*dst = NULL; *one = false;
	uint64_t per = im.ri ? (uint64_t)im.ri * im.nblk : (uint64_t)im.nmcu * im.nblk;
	uint64_t k = u / per, j = u % per;
	if (k >= nint) return JPEGQS_DECODE_UNITS;
	uint32_t b0 = ivstart[k], b1 = k + 1 < nint ? ivstart[k + 1] : nbytes;
	uint64_t bit = 8ull * b0 + j;
	uint32_t err = 0;
	if (bit >= 8ull * b1) err |= JPEGQS_DECODE_TRUNCATED;
	else *one = unst[bit >> 3] >> (7 - (bit & 7)) & 1;
	uint32_t kk = (uint32_t)(u % im.nblk), c = im.u_comp[kk]; uint64_t m = u / im.nblk;
	uint64_t bx = (uint64_t)(m % im.nx) * im.u_hs[kk] + im.u_h[kk], by = (uint64_t)(m / im.nx) * im.u_vs[kk] + im.u_v[kk];
	if (bx < im.wblk[c] && by < im.hblk[c]) *dst = im.coef[c] + ((size_t)by * im.wblk[c] + bx) * 64;
	return err;
}

HD static inline bool qs_first(uint32_t kind) { return kind <= QS_ACF; }

/* ---------------------------------------------------------------- kernels */
struct QsPtrs { char *base; uint32_t n, pad; uint64_t off[QS_GROUP_SEGS]; };
#define QS_SEG(P, i) (*reinterpret_cast<const QsSeg *>((P).base + (P).off[i]))

struct QsZeroPack { int4 *p[QS_GROUP_IMGS * 4]; uint64_t n16[QS_GROUP_IMGS * 4]; int32_t *status[QS_GROUP_IMGS]; int narr, nimg; };

/* blockIdx.y = array: zeroes the output arrays; block (0, 0) the images' status words */
__global__ void __launch_bounds__(256) qs_zero_kernel(const __grid_constant__ QsZeroPack z) {
	if (blockIdx.x == 0 && blockIdx.y == 0 && (int)threadIdx.x < z.nimg) *z.status[threadIdx.x] = 0;
	if ((int)blockIdx.y >= z.narr) return;
	int4 *p = z.p[blockIdx.y];
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < z.n16[blockIdx.y]; i += (uint64_t)gridDim.x * blockDim.x)
		p[i] = make_int4(0, 0, 0, 0);
}

struct QsStorePack {
	QsSeg seg[QS_PACK];
	int8_t slot[QS_PACK][8];           /* table t of scan j: pool index, -1 = not used */
	uint8_t bits[QS_PACK_TABS][17], val[QS_PACK_TABS][256];
	int n;
};
static_assert(sizeof(QsStorePack) <= 32000, "QsStorePack exceeds the kernel parameter space");

/* blockIdx.x = scan, threadIdx.x = table slot: derived tables, descriptor, state */
__global__ void qs_store_kernel(const __grid_constant__ QsStorePack p) {
	int j = blockIdx.x, t = threadIdx.x;
	if (j >= p.n || t >= 8) return;
	const QsSeg &s = p.seg[j];
	if (p.slot[j][t] >= 0) qd_build(s.im.tab + t, p.bits[p.slot[j][t]], p.val[p.slot[j][t]]);
	if (t == 0) {
		*reinterpret_cast<QsSeg *>(reinterpret_cast<char *>(s.im.tab) - 2048) = s;
		memset(s.im.st, 0, sizeof(QdState));
	}
}

__global__ void __launch_bounds__(QD_BT) qs_scan_kernel(const __grid_constant__ QsPtrs P) {
	if (blockIdx.y >= P.n) return;
	qd_scan_body(QS_SEG(P, blockIdx.y).im, blockIdx.x);
}
__global__ void __launch_bounds__(QD_SCAN_T) qs_seg_kernel(const __grid_constant__ QsPtrs P) {
	if (blockIdx.x >= P.n) return;
	qd_seg_body(QS_SEG(P, blockIdx.x).im);
}
__global__ void __launch_bounds__(QD_BT) qs_compact_kernel(const __grid_constant__ QsPtrs P) {
	if (blockIdx.y >= P.n) return;
	qd_compact_body(QS_SEG(P, blockIdx.y).im, blockIdx.x);
}
__global__ void __launch_bounds__(QD_SCAN_T) qs_iv_kernel(const __grid_constant__ QsPtrs P) {
	if (blockIdx.x >= P.n || !qs_first(QS_SEG(P, blockIdx.x).kind)) return;
	qd_iv_body(QS_SEG(P, blockIdx.x).im);
}

/* qd_sync_kernel over first scans */
__global__ void __launch_bounds__(QD_ST) qs_sync_kernel(const __grid_constant__ QsPtrs P, int mode) {
	if (blockIdx.y >= P.n) return;
	const QsSeg &sg = QS_SEG(P, blockIdx.y);
	const QdImg &im = sg.im;
	if (!qs_first(sg.kind)) return;
	const QdState *st = im.st;
	uint32_t nsub = st->nsub, s = blockIdx.x * QD_ST + threadIdx.x;
	if (blockIdx.x * QD_ST >= nsub) return;
	__shared__ uint64_t s_exit[QD_ST];
	QsView v;
	qs_view(sg, im.tab, im.unst, st->nbytes, &v);
	bool act = s < nsub;
	QdSpan sp = {};
	QdSub me = {};
	me.entry = QD_NONE;
	if (act) {
		sp = qd_span(im, im.ivstart, im.ivsub0, st->nint, st->nbytes, nsub, s);
		v.rd.lim = (uint32_t)(sp.iv_end >> 3);
		if (mode == 0) {
			qs_path(v, sp.begin << 4, sp.end, sp.iv_end, sp.last, NULL, &me);
			me.iv = sp.iv; me.sync_units = 0;
		} else me = im.sub[s];
	}
	for (;;) {
		s_exit[threadIdx.x] = me.exit;
		__syncthreads();
		bool changed = false;
		if (act && !sp.first) {
			uint64_t want;
			if (threadIdx.x > 0) want = s_exit[threadIdx.x - 1];
			/* as in qd_sync_kernel: a stale read of the previous block's record costs a re-decode only */
			else if (mode == 1) want = *(volatile const uint64_t *)&im.sub[s - 1].exit;
			else want = me.entry;
			if (want != me.entry) {
				QdSub nw = me;
				nw.sync_units += qs_path(v, want, sp.end, sp.iv_end, sp.last, &me, &nw);
				me = nw; changed = true;
			}
		}
		if (!__syncthreads_or(changed)) break;
		mode = mode == 1 ? 2 : mode;
	}
	if (act) im.sub[s] = me;
}

/* qd_chain_kernel over first scans */
__global__ void __launch_bounds__(32) qs_chain_kernel(const __grid_constant__ QsPtrs P) {
	if (blockIdx.x >= P.n) return;
	const QsSeg &sg = QS_SEG(P, blockIdx.x);
	const QdImg &im = sg.im;
	if (!qs_first(sg.kind)) return;
	const QdState *st = im.st;
	uint32_t nsub = st->nsub, lane = threadIdx.x;
	QsView v;
	qs_view(sg, im.tab, im.unst, st->nbytes, &v);
	for (uint32_t base = 1; base < nsub; ) {
		uint32_t s = base + lane;
		bool bad = false;
		if (s < nsub) {
			uint64_t e = ((volatile QdSub *)im.sub)[s].entry, x = ((volatile QdSub *)im.sub)[s - 1].exit;
			bad = e != x && im.sub[s].iv == im.sub[s - 1].iv;
		}
		uint32_t m = __ballot_sync(0xFFFFFFFFu, bad);
		if (!m) { base += 32; continue; }
		uint32_t f = base + __ffs(m) - 1;
		if (lane == 0) {
			QdSpan sp = qd_span(im, im.ivstart, im.ivsub0, st->nint, st->nbytes, nsub, f);
			QsView w = v;
			w.rd.lim = (uint32_t)(sp.iv_end >> 3);
			QdSub old = im.sub[f], nw = old;
			nw.sync_units += qs_path(w, im.sub[f - 1].exit, sp.end, sp.iv_end, sp.last, &old, &nw);
			im.sub[f] = nw;
			__threadfence_block();
		}
		__syncwarp();
		base = f + 1;
	}
}

/* the checks of a placed subsequence (place kernel and model) */
HD static inline uint32_t qs_place_check(const QsSeg &sg, const QdSub &sb, const QdSpan &sp, uint64_t g0, uint64_t total,
		uint32_t nint) {
	const QdImg &im = sg.im;
	uint32_t bad = 0;
	if (sb.entry == QD_NONE) bad |= JPEGQS_DECODE_UNITS;
	if (sb.err) bad |= (uint32_t)(sb.err & 0xFF);
	if (sb.entry != QD_NONE && (uint32_t)(sb.entry & 15) != g0 % im.period) bad |= JPEGQS_DECODE_UNITS;
	if (g0 > total) bad |= JPEGQS_DECODE_UNITS;
	if (sp.last) {
		int64_t want = qd_expect(im, sp.iv, nint), got = (int64_t)(g0 + sb.cnt);
		/* an AC first scan's last end-of-band run may reach past the interval: libjpeg cuts it */
		if (sg.kind == QS_ACF ? got < want : got != want) bad |= JPEGQS_DECODE_UNITS;
		if ((sb.exit >> 4) > sp.iv_end) bad |= JPEGQS_DECODE_TRUNCATED;
	}
	return bad;
}

struct QsAcc { uint32_t flag; uint64_t cnt; };
struct QsDc { uint32_t flag; int32_t v[4]; };
__global__ void __launch_bounds__(QD_SCAN_T) qs_place_kernel(const __grid_constant__ QsPtrs P) {
	if (blockIdx.x >= P.n) return;
	const QsSeg &sg = QS_SEG(P, blockIdx.x);
	const QdImg &im = sg.im;
	if (!qs_first(sg.kind)) return;
	const QdState *st = im.st;
	typedef cub::BlockScan<QsAcc, QD_SCAN_T> S1;
	typedef cub::BlockScan<QsDc, QD_SCAN_T> S2;
	__shared__ union { typename S1::TempStorage a; typename S2::TempStorage b; } tmp;
	struct Op1 { __device__ QsAcc operator()(QsAcc a, QsAcc b) const { return b.flag ? b : QsAcc{ a.flag, a.cnt + b.cnt }; } };
	struct Op2 { __device__ QsDc operator()(QsDc a, QsDc b) const {
		if (b.flag) return b;
		QsDc r; r.flag = a.flag; for (int c = 0; c < 4; c++) r.v[c] = a.v[c] + b.v[c]; return r; } };
	uint32_t nsub = st->nsub, nint = st->nint;
	uint64_t total = (uint64_t)im.nmcu * im.nblk;
	QsAcc c1 = { 1, 0 };
	QsDc c2 = { 1, { 0, 0, 0, 0 } };
	uint32_t bad = 0;
	for (uint32_t base = 0; base < nsub; base += QD_SCAN_T) {
		uint32_t s = base + threadIdx.x;
		bool act = s < nsub;
		QdSub sb = {};
		QdSpan sp = {};
		if (act) { sb = im.sub[s]; sp = qd_span(im, im.ivstart, im.ivsub0, nint, st->nbytes, nsub, s); }
		QsAcc a = { act && sp.first ? 1u : 0u, act ? (uint64_t)sb.cnt : 0ull }, ae, aagg;
		S1(tmp.a).ExclusiveScan(a, ae, c1, Op1(), aagg);
		__syncthreads();
		uint64_t g0 = a.flag ? 0 : ae.cnt;
		QsDc d = { a.flag, { 0, 0, 0, 0 } };
		if (act) for (uint32_t r = 0; r < im.nblk; r++) d.v[im.u_comp[(g0 + r) % im.nblk]] += sb.dcs[r];
		QsDc de, dagg;
		S2(tmp.b).ExclusiveScan(d, de, c2, Op2(), dagg);
		__syncthreads();
		if (act) {
			QdSub &w = im.sub[s];
			w.g0 = (uint32_t)(g0 > total ? total : g0);
			for (int c = 0; c < 4; c++) w.pred[c] = d.flag ? 0 : de.v[c];
			bad |= qs_place_check(sg, sb, sp, g0, total, nint);
		}
		c1 = Op1()(c1, aagg);
		c2 = Op2()(c2, dagg);
		__syncthreads();
	}
	if (nsub < nint) bad |= JPEGQS_DECODE_UNITS;
	if (bad) atomicOr(im.status, (int)bad);
}

__global__ void __launch_bounds__(QD_ST) qs_final_kernel(const __grid_constant__ QsPtrs P) {
	if (blockIdx.y >= P.n) return;
	const QsSeg &sg = QS_SEG(P, blockIdx.y);
	const QdImg &im = sg.im;
	if (!qs_first(sg.kind)) return;
	const QdState *st = im.st;
	uint32_t s = blockIdx.x * QD_ST + threadIdx.x;
	if (s >= st->nsub) return;
	QsView v;
	qs_view(sg, im.tab, im.unst, st->nbytes, &v);
	QdSub sb = im.sub[s];
	uint32_t nint = st->nint;
	v.rd.lim = sb.iv + 1 < nint ? im.ivstart[sb.iv + 1] : st->nbytes;
	for (uint32_t k = 0; k < im.nblk && k < QD_MAX_UNITS; k++) { v.dc[k] = im.tab + im.u_dc[k]; v.ac[k] = im.tab + 4 + im.u_ac[k]; }
	v.period = im.nblk;
	uint32_t e = qs_final_sub(sg, v, sb, nint);
	if (e) atomicOr(im.status, (int)e);
}

/* every DC refinement scan of the group: one thread per block */
__global__ void __launch_bounds__(256) qs_dcr_kernel(const __grid_constant__ QsPtrs P) {
	if (blockIdx.y >= P.n) return;
	const QsSeg &sg = QS_SEG(P, blockIdx.y);
	const QdImg &im = sg.im;
	if (sg.kind != QS_DCR) return;
	uint64_t u = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	uint32_t e = 0;
	if (u < (uint64_t)im.nmcu * im.nblk) {
		const QdState *st = im.st;
		int16_t *dst; bool one;
		e = qs_dcr_unit(sg, im.unst, im.ivstart, st->nint, st->nbytes, u, &dst, &one);
		/* blocks are 128-byte aligned: blk[0] is the low half of its 32-bit word */
		if (dst && one) atomicOr(reinterpret_cast<unsigned int *>(dst), 1u << sg.Al);
	}
	e = __reduce_or_sync(0xFFFFFFFFu, e);
	if (e && (threadIdx.x & 31) == 0) atomicOr(im.status, (int)e);
}

/* the AC refinement scans of one level: one restart interval per warp, decoded by its lane 0.  The
 * decode of an interval is serial; a warp of its own keeps the intervals' divergent decoders apart
 * and spreads them over the SMs (QS_RT / 32 intervals per block). */
__global__ void __launch_bounds__(QS_RT) qs_acr_kernel(const __grid_constant__ QsPtrs P, uint32_t level) {
	if (blockIdx.y >= P.n) return;
	const QsSeg &sg = QS_SEG(P, blockIdx.y);
	const QdImg &im = sg.im;
	if (sg.kind != QS_ACR || sg.level != level) return;
	const QdState *st = im.st;
	uint32_t nint = st->nint;
	if (blockIdx.x * (QS_RT / 32) >= nint) return;
	__shared__ uint64_t tab[8][256];
	for (int i = threadIdx.x; i < 8 * 256; i += QS_RT) tab[i >> 8][i & 255] = qs_zz_entry(i >> 8, i & 255);
	__syncthreads();
	uint32_t k = blockIdx.x * (QS_RT / 32) + threadIdx.x / 32;
	if (k >= nint || (threadIdx.x & 31)) return;
	uint32_t b0 = im.ivstart[k], b1 = k + 1 < nint ? im.ivstart[k + 1] : st->nbytes;
	if (b1 < b0) b1 = b0;
	uint64_t u0 = (uint64_t)k * im.ri, nu = (uint64_t)qd_expect(im, k, nint);
	uint32_t e = qs_acr_interval(sg, im.tab + 4 + im.u_ac[0], im.unst, b0, b1, u0, nu, tab);
	if (e) atomicOr(im.status, (int)e);
}

/* ---------------------------------------------------------------- host: checks, workspace, launches */
struct jpegqs_cuda_ctx;
void qs_ctx_decode_info(jpegqs_cuda_ctx *ctx, int *device, cudaStream_t *stream, int *sub_bytes);
void qs_ctx_decode_done(jpegqs_cuda_ctx *ctx, int launches, const char *err);
extern "C" void qs_set_host_error(const char *msg);

static size_t qs_a256(size_t x) { return (x + 255) & ~(size_t)255; }

struct QsPlan {                        /* one scan, host side */
	QsSeg seg;
	uint8_t bits[8][17], val[8][256];  /* bits[t][0] = 1: table t used */
	size_t bytes, nsub_grid;
};

/* the image checks of decode_async */
static const char *qs_check_image(const jpegqs_cuda_image *im, bool ptrs) {
	int nc = im->ncomp, maxh = 1, maxv = 1;
	if (nc < 1 || nc > 4) return "ncomp outside 1..4";
	for (int c = 0; c < nc; c++) {
		const jpegqs_cuda_comp &cc = im->comp[c];
		if (cc.h_samp < 1 || cc.h_samp > 4 || cc.v_samp < 1 || cc.v_samp > 4) return "sampling factor outside 1..4";
		if (cc.rows || cc.rows_up) return "rows / rows_up set";
		if (ptrs && !cc.coef) return "coef NULL";
		if (ptrs && ((uintptr_t)cc.coef & 15)) return "coef not 16-byte aligned";
		maxh = cc.h_samp > maxh ? cc.h_samp : maxh; maxv = cc.v_samp > maxv ? cc.v_samp : maxv;
	}
	for (int c = 0; c < nc; c++) {
		const jpegqs_cuda_comp &cc = im->comp[c];
		uint64_t wb = ((uint64_t)im->image_width * cc.h_samp + 8 * maxh - 1) / (8 * maxh);
		uint64_t hb = ((uint64_t)im->image_height * cc.v_samp + 8 * maxv - 1) / (8 * maxv);
		if (!im->image_width || !im->image_height || cc.wblk != wb || cc.hblk != hb) return "wblk / hblk are not libjpeg's for this image size";
	}
	return NULL;
}

/* checks scan j of an image (image already checked) and fills its plan */
static const char *qs_check_scan(const jpegqs_cuda_image *im, const jpegqs_cuda_scan_rec *sc, size_t len, int sub_bytes,
		QsPlan *pl) {
	memset(pl, 0, sizeof(*pl));
	QsSeg &s = pl->seg;
	QdImg &d = s.im;
	int nc = im->ncomp, maxh = 1, maxv = 1, seen = 0;
	for (int c = 0; c < nc; c++) {
		maxh = im->comp[c].h_samp > maxh ? im->comp[c].h_samp : maxh; maxv = im->comp[c].v_samp > maxv ? im->comp[c].v_samp : maxv;
		d.wblk[c] = im->comp[c].wblk; d.hblk[c] = im->comp[c].hblk; d.coef[c] = im->comp[c].coef;
	}
	if (sc->sof != 0xC0 && sc->sof != 0xC1 && sc->sof != 0xC2) return "sof not 0xC0 / 0xC1 / 0xC2";
	bool prog = sc->sof == 0xC2;
	if (sc->ncomp < 1 || sc->ncomp > nc) return "scan ncomp outside 1..frame components";
	for (int k = 0; k < sc->ncomp; k++) {
		int c = sc->comp[k];
		if (c < 0 || c >= nc || (seen >> c & 1)) return "scan components are not distinct frame components";
		seen |= 1 << c;
		if (sc->dc_tbl[k] < 0 || sc->dc_tbl[k] > 3 || sc->ac_tbl[k] < 0 || sc->ac_tbl[k] > 3) return "a selector outside 0..3";
	}
	if (prog) {
		if (sc->Ss < 0 || sc->Ss > 63 || sc->Se < sc->Ss || sc->Se > 63 || sc->Ah < 0 || sc->Ah > 13 || sc->Al < 0 || sc->Al > 13)
			return "Ss / Se / Ah / Al outside T.81's ranges";
		if (sc->Ss > 0 && sc->ncomp != 1) return "an AC scan of several components";
		s.kind = sc->Ss == 0 ? (sc->Ah ? QS_DCR : QS_DCF) : (sc->Ah ? QS_ACR : QS_ACF);
	} else {
		if (sc->Ss != 0 || sc->Se != 63 || sc->Ah != 0 || sc->Al != 0) return "a sequential scan with Ss / Se / Ah / Al other than 0 / 63 / 0 / 0";
		s.kind = QS_SEQ;
	}
	s.Ss = (uint32_t)sc->Ss; s.Se = (uint32_t)sc->Se; s.Al = (uint32_t)sc->Al;
	if (sc->offset >= sc->end || sc->end > len) return "offset / end outside the data";
	if (sc->end - sc->offset > 0xFFFFFFF0ull) return "entropy-coded data longer than 4 GB";
	if (sc->restart_interval > 65535) return "restart interval beyond 65535";
	bool need_dc = s.kind == QS_SEQ || s.kind == QS_DCF, need_ac = s.kind == QS_SEQ || s.kind == QS_ACF || s.kind == QS_ACR;
	for (int t = 0; t < 8; t++) {
		int dc = t < 4, j = t & 3, used = 0;
		if (dc ? !need_dc : !need_ac) continue;
		for (int k = 0; k < sc->ncomp; k++) used |= dc ? sc->dc_tbl[k] == j : sc->ac_tbl[k] == j;
		if (!used) continue;
		if (!(dc ? sc->dc_present[j] : sc->ac_present[j])) return "a selector names an absent table";
		memcpy(pl->bits[t], dc ? sc->dc_bits[j] : sc->ac_bits[j], 17);
		memcpy(pl->val[t], dc ? sc->dc_val[j] : sc->ac_val[j], 256);
		pl->bits[t][0] = 1;
		QdHuff h;
		if (qd_build(&h, pl->bits[t], pl->val[t])) return "a selected Huffman table is invalid";
		if (dc) { int n = 0; for (int l = 1; l <= 16; l++) n += pl->bits[t][l]; for (int i = 0; i < n; i++) if (pl->val[t][i] > 15) return "a DC table holds a symbol > 15"; }
	}
	/* the units of one MCU (A.2.3; one component: not interleaved, one block) */
	uint32_t nb = 0;
	if (sc->ncomp == 1) {
		int c = sc->comp[0];
		d.nx = d.wblk[c]; d.ny = d.hblk[c];
		d.u_comp[0] = (uint8_t)c; d.u_hs[0] = d.u_vs[0] = 1; d.u_h[0] = d.u_v[0] = 0;
		d.u_dc[0] = (uint8_t)sc->dc_tbl[0]; d.u_ac[0] = (uint8_t)sc->ac_tbl[0];
		nb = 1;
	} else {
		d.nx = (uint32_t)(((uint64_t)im->image_width + 8 * maxh - 1) / (8 * maxh));
		d.ny = (uint32_t)(((uint64_t)im->image_height + 8 * maxv - 1) / (8 * maxv));
		for (int k = 0; k < sc->ncomp; k++) {
			const jpegqs_cuda_comp &cc = im->comp[sc->comp[k]];
			for (int v = 0; v < cc.v_samp; v++) for (int h = 0; h < cc.h_samp; h++) {
				if (nb >= QD_MAX_UNITS) return "more than 10 blocks per MCU";
				d.u_comp[nb] = (uint8_t)sc->comp[k]; d.u_h[nb] = (uint8_t)h; d.u_v[nb] = (uint8_t)v;
				d.u_hs[nb] = (uint8_t)cc.h_samp; d.u_vs[nb] = (uint8_t)cc.v_samp;
				d.u_dc[nb] = (uint8_t)sc->dc_tbl[k]; d.u_ac[nb] = (uint8_t)sc->ac_tbl[k];
				nb++;
			}
		}
	}
	d.nblk = nb;
	uint64_t nmcu = (uint64_t)d.nx * d.ny;
	if (nmcu * nb > 0xFFFFFFF0ull) return "image too large";
	d.nmcu = (uint32_t)nmcu;
	/* the smallest period of the units' table sequence (the tables the scan decodes with) */
	for (d.period = 1; d.period < nb; d.period++) {
		if (nb % d.period) continue;
		uint32_t k;
		for (k = d.period; k < nb; k++) {
			int a = d.u_dc[k], b = d.u_dc[k - d.period], x = 4 + d.u_ac[k], y = 4 + d.u_ac[k - d.period];
			if (need_dc && (memcmp(pl->bits[a], pl->bits[b], 17) || memcmp(pl->val[a], pl->val[b], 256))) break;
			if (need_ac && (memcmp(pl->bits[x], pl->bits[y], 17) || memcmp(pl->val[x], pl->val[y], 256))) break;
		}
		if (k == nb) break;
	}
	d.ri = sc->restart_interval;
	d.nint_cap = d.ri ? (uint32_t)((nmcu + d.ri - 1) / d.ri) : 1;
	if (!d.nint_cap) d.nint_cap = 1;
	uint64_t L = sc->end - sc->offset;
	d.off = sc->offset; d.len = sc->end;
	d.nchunk = (uint32_t)((L + QD_CHUNK - 1) / QD_CHUNK);
	d.sub_bytes = (uint32_t)sub_bytes;
	bool first = qs_first(s.kind);
	d.nsub_cap = first ? (uint32_t)(L / QD_SUB_MIN + d.nint_cap) : 0;
	pl->nsub_grid = first ? L / (uint64_t)sub_bytes + d.nint_cap : 0;
	pl->bytes = QD_FIXED + qs_a256(L + 8) + qs_a256(24 * (size_t)d.nchunk) + 2 * qs_a256(4 * (size_t)d.nint_cap) +
		(first ? qs_a256(96 * (size_t)d.nsub_cap) : 0);
	return NULL;
}

/* AC refinement levels of one image's scans: one more than the highest among earlier AC refinement
 * scans of the same component whose bands overlap */
static void qs_levels(std::vector<QsPlan> &pl, size_t first, size_t n) {
	for (size_t j = first; j < first + n; j++) {
		QsSeg &b = pl[j].seg;
		if (b.kind != QS_ACR) continue;
		uint32_t lv = 0;
		for (size_t i = first; i < j; i++) {
			const QsSeg &a = pl[i].seg;
			if (a.kind == QS_ACR && a.im.u_comp[0] == b.im.u_comp[0] && a.Ss <= b.Se && b.Ss <= a.Se && a.level + 1 > lv) lv = a.level + 1;
		}
		b.level = lv;
	}
}

static void qs_carve(QsPlan *pl, char *w, int32_t *status) {
	QdImg &d = pl->seg.im;
	uint64_t L = d.len - d.off;
	d.st = reinterpret_cast<QdState *>(w + 1024);
	d.tab = reinterpret_cast<QdHuff *>(w + 2048);
	w += QD_FIXED;
	d.unst = reinterpret_cast<uint8_t *>(w); w += qs_a256(L + 8);
	d.chunk = reinterpret_cast<QdChunk *>(w); w += qs_a256(24 * (size_t)d.nchunk);
	d.ivstart = reinterpret_cast<uint32_t *>(w); w += qs_a256(4 * (size_t)d.nint_cap);
	d.ivsub0 = reinterpret_cast<uint32_t *>(w); w += qs_a256(4 * (size_t)d.nint_cap);
	d.sub = reinterpret_cast<QdSub *>(w);
	d.status = status;
}

/* checks every image and scan; fills plans (per scan, image after image) and first[i] */
static const char *qs_plan_all(int n, const jpegqs_cuda_image *imgs, const jpegqs_cuda_scan_rec *const *scans, const int *nscans,
		const size_t *data_len, bool ptrs, int sub_bytes, std::vector<QsPlan> &plan, std::vector<size_t> &first, int *bad_img,
		size_t *total) {
	*total = 0;
	for (int i = 0; i < n; i++) {
		*bad_img = i;
		const char *e = qs_check_image(&imgs[i], ptrs);
		if (e) return e;
		if (nscans[i] < 1 || nscans[i] > JPEGQS_MAX_SCANS) return "nscans outside 1..64";
		if (!scans[i]) return "scans entry NULL";
		first.push_back(plan.size());
		for (int j = 0; j < nscans[i]; j++) {
			plan.emplace_back();
			e = qs_check_scan(&imgs[i], &scans[i][j], data_len[i], sub_bytes, &plan.back());
			if (e) return e;
			*total += plan.back().bytes;
		}
		qs_levels(plan, first.back(), (size_t)nscans[i]);
	}
	first.push_back(plan.size());
	return NULL;
}

extern "C" int jpegqs_cuda_decode_scans_workspace_bytes(int n, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_scan_rec *const *scans, const int *nscans, const size_t *data_len, size_t *bytes) {
	if (n < 0 || !bytes || (n && (!imgs || !scans || !nscans || !data_len))) { qs_set_host_error("jpegqs_cuda_decode_scans_workspace_bytes: NULL argument"); return JPEGQS_ERR_ARG; }
	std::vector<QsPlan> plan; std::vector<size_t> first; int bad = 0; size_t total = 0;
	const char *e = qs_plan_all(n, imgs, scans, nscans, data_len, false, QD_SUB_MIN, plan, first, &bad, &total);
	if (e) { char m[256]; snprintf(m, sizeof(m), "jpegqs_cuda_decode_scans_workspace_bytes: image %d: %s", bad, e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
	*bytes = total;
	return 0;
}

#define QS_CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	snprintf(msg, sizeof(msg), "%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
	qs_ctx_decode_done(ctx, launches, msg); return JPEGQS_ERR_CUDA; } } while (0)

extern "C" int jpegqs_cuda_decode_scans_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_scan_rec *const *scans, const int *nscans, const uint8_t *const *data_dev,
		const size_t *data_len, void *workspace, size_t workspace_bytes, int32_t *status_dev, void *stream) {
	char msg[512] = "";
	int launches = 0;
	if (!ctx) return JPEGQS_ERR_ARG;
	int device, sub_bytes; cudaStream_t st;
	qs_ctx_decode_info(ctx, &device, &st, &sub_bytes);
	if (stream) st = (cudaStream_t)stream;
	if (n < 0 || (n && (!imgs || !scans || !nscans || !data_dev || !data_len || !status_dev || !workspace))) {
		qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_decode_scans_async: NULL argument"); return JPEGQS_ERR_ARG;
	}
	if ((uintptr_t)workspace & 255) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_decode_scans_async: workspace not 256-byte aligned"); return JPEGQS_ERR_ARG; }
	for (int i = 0; i < n; i++)
		if (!data_dev[i]) { snprintf(msg, sizeof(msg), "jpegqs_cuda_decode_scans_async: image %d: data_dev entry NULL", i); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
	std::vector<QsPlan> plan; std::vector<size_t> first; int bad = 0; size_t need = 0;
	const char *e = qs_plan_all(n, imgs, scans, nscans, data_len, true, sub_bytes, plan, first, &bad, &need);
	if (e) { snprintf(msg, sizeof(msg), "jpegqs_cuda_decode_scans_async: image %d: %s", bad, e); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
	if (workspace_bytes < need) {
		snprintf(msg, sizeof(msg), "jpegqs_cuda_decode_scans_async: workspace of %zu bytes, %zu needed", workspace_bytes, need);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (!n) { qs_ctx_decode_done(ctx, 0, ""); return 0; }
	QS_CK(cudaSetDevice(device));
	char *w = (char *)workspace;
	for (int i = 0; i < n; i++)
		for (size_t j = first[i]; j < first[i + 1]; j++) {
			plan[j].seg.im.data = data_dev[i];
			qs_carve(&plan[j], w, status_dev + i); w += plan[j].bytes;
		}
	std::unique_ptr<QsStorePack> hold(new QsStorePack());         /* 25 KB: not on the stack */
	std::unique_ptr<QsPtrs> hp(new QsPtrs());
	for (int g0 = 0; g0 < n; ) {
		int g = 0;                                                   /* images of this group */
		while (g0 + g < n && g < QS_GROUP_IMGS && first[g0 + g + 1] - first[g0] <= QS_GROUP_SEGS) g++;
		size_t s0 = first[g0], s1 = first[g0 + g];
		/* zero the arrays and the status words */
		QsZeroPack z;
		memset(&z, 0, sizeof(z));
		uint64_t maxz = 1;
		for (int i = 0; i < g; i++) {
			const jpegqs_cuda_image &im = imgs[g0 + i];
			z.status[z.nimg++] = status_dev + g0 + i;
			for (int c = 0; c < im.ncomp; c++) {
				z.p[z.narr] = reinterpret_cast<int4 *>(im.comp[c].coef);
				z.n16[z.narr] = (uint64_t)im.comp[c].wblk * im.comp[c].hblk * 8;
				maxz = std::max(maxz, z.n16[z.narr]);
				z.narr++;
			}
		}
		uint32_t zx = (uint32_t)std::min<uint64_t>((maxz + 255) / 256, 1024);
		qs_zero_kernel<<<dim3(zx, std::max(z.narr, 1)), 256, 0, st>>>(z); launches++;
		/* descriptors and tables: store launches of up to QS_PACK scans and QS_PACK_TABS tables */
		QsStorePack &pack = *hold;
		for (size_t j = s0; j < s1; ) {
			memset(&pack, 0, sizeof(pack));
			int nt = 0;
			while (j < s1 && pack.n < QS_PACK) {
				const QsPlan &pl = plan[j];
				int used = 0;
				for (int t = 0; t < 8; t++) used += pl.bits[t][0] == 1;
				if (nt + used > QS_PACK_TABS) break;
				pack.seg[pack.n] = pl.seg;
				for (int t = 0; t < 8; t++) {
					pack.slot[pack.n][t] = -1;
					if (pl.bits[t][0] != 1) continue;
					memcpy(pack.bits[nt], pl.bits[t], 17); memcpy(pack.val[nt], pl.val[t], 256);
					pack.slot[pack.n][t] = (int8_t)nt++;
				}
				pack.n++; j++;
			}
			qs_store_kernel<<<pack.n, 32, 0, st>>>(pack); launches++;
		}
		QsPtrs &P = *hp;
		memset(&P, 0, sizeof(P));
		P.base = (char *)workspace; P.n = (uint32_t)(s1 - s0);
		uint32_t maxchunk = 1, maxlevel = 0; size_t maxsub = 1; uint64_t maxdcr = 0, maxint = 1;
		bool any_first = false, any_acr = false;
		for (size_t j = s0; j < s1; j++) {
			const QsPlan &pl = plan[j];
			P.off[j - s0] = (uint64_t)(reinterpret_cast<const char *>(pl.seg.im.tab) - 2048 - (const char *)workspace);
			maxchunk = std::max(maxchunk, pl.seg.im.nchunk);
			maxsub = std::max(maxsub, pl.nsub_grid);
			any_first |= qs_first(pl.seg.kind);
			if (pl.seg.kind == QS_DCR) maxdcr = std::max(maxdcr, (uint64_t)pl.seg.im.nmcu * pl.seg.im.nblk);
			if (pl.seg.kind == QS_ACR) { any_acr = true; maxlevel = std::max(maxlevel, pl.seg.level); maxint = std::max(maxint, (uint64_t)pl.seg.im.nint_cap); }
		}
		uint32_t ns = P.n, subblocks = (uint32_t)((maxsub + QD_ST - 1) / QD_ST);
		qs_scan_kernel<<<dim3(maxchunk, ns), QD_BT, 0, st>>>(P); launches++;
		qs_seg_kernel<<<ns, QD_SCAN_T, 0, st>>>(P); launches++;
		qs_compact_kernel<<<dim3(maxchunk, ns), QD_BT, 0, st>>>(P); launches++;
		if (any_first) {
			qs_iv_kernel<<<ns, QD_SCAN_T, 0, st>>>(P); launches++;
			qs_sync_kernel<<<dim3(subblocks, ns), QD_ST, 0, st>>>(P, 0); launches++;
			qs_sync_kernel<<<dim3(subblocks, ns), QD_ST, 0, st>>>(P, 1); launches++;
			qs_chain_kernel<<<ns, 32, 0, st>>>(P); launches++;
			qs_place_kernel<<<ns, QD_SCAN_T, 0, st>>>(P); launches++;
			qs_final_kernel<<<dim3(subblocks, ns), QD_ST, 0, st>>>(P); launches++;
		}
		if (maxdcr) { qs_dcr_kernel<<<dim3((uint32_t)((maxdcr + 255) / 256), ns), 256, 0, st>>>(P); launches++; }
		if (any_acr)
			for (uint32_t lv = 0; lv <= maxlevel; lv++) {
				qs_acr_kernel<<<dim3((uint32_t)((maxint + QS_RT / 32 - 1) / (QS_RT / 32)), ns), QS_RT, 0, st>>>(P, lv); launches++;
			}
		QS_CK(cudaGetLastError());
		g0 += g;
	}
	qs_ctx_decode_done(ctx, launches, "");
	return 0;
}

/* ---------------------------------------------------------------- the CPU model */
extern "C" int jpegqs_cuda_decode_scans_model(const jpegqs_cuda_image *img, const jpegqs_cuda_scan_rec *scans, int nscans,
		const uint8_t *data, size_t data_len, int sub_bytes, int32_t *status) {
	if (!img || !scans || !data || !status) { qs_set_host_error("jpegqs_cuda_decode_scans_model: NULL argument"); return JPEGQS_ERR_ARG; }
	if (sub_bytes < QD_SUB_MIN) { qs_set_host_error("jpegqs_cuda_decode_scans_model: sub_bytes below 32"); return JPEGQS_ERR_ARG; }
	std::vector<QsPlan> plan; std::vector<size_t> first; int bad = 0; size_t total = 0;
	const jpegqs_cuda_scan_rec *sp0 = scans;
	const char *e = qs_plan_all(1, img, &sp0, &nscans, &data_len, true, sub_bytes, plan, first, &bad, &total);
	if (e) { char m[256]; snprintf(m, sizeof(m), "jpegqs_cuda_decode_scans_model: %s", e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
	for (int c = 0; c < img->ncomp; c++) memset(img->comp[c].coef, 0, (size_t)img->comp[c].wblk * img->comp[c].hblk * 128);
	uint64_t zz[8][256];
	for (int r = 0; r < 8; r++) for (int b = 0; b < 256; b++) zz[r][b] = qs_zz_entry(r, b);
	uint32_t stat = 0;
	struct Seg { std::vector<QdHuff> tab; std::vector<uint8_t> unst; std::vector<uint32_t> ivstart; uint32_t nbytes, nint; };
	std::vector<Seg> sd(plan.size());
	/* bytes: every scan */
	for (size_t j = 0; j < plan.size(); j++) {
		QdImg &im = plan[j].seg.im;
		Seg &s = sd[j];
		im.data = data;
		s.tab.resize(8);
		for (int t = 0; t < 8; t++) if (plan[j].bits[t][0] == 1) qd_build(&s.tab[t], plan[j].bits[t], plan[j].val[t]);
		s.ivstart.assign(im.nint_cap, 0);
		uint32_t nrst = 0;
		bool ri = im.ri != 0;
		for (uint64_t p = im.off; p < im.len; p++) {
			bool t, k, r;
			qd_byte_class(data, im.off, im.len, p, ri, &t, &k, &r);
			if (t) break;
			if (r) {
				if ((uint32_t)(data[p + 1] & 7) != (nrst & 7)) stat |= JPEGQS_DECODE_RESTART;
				if (nrst + 1 < im.nint_cap) s.ivstart[nrst + 1] = (uint32_t)s.unst.size();
				nrst++;
			}
			if (k) s.unst.push_back(data[p]);
		}
		s.nbytes = (uint32_t)s.unst.size();
		s.nint = im.ri ? nrst + 1 : 1;
		if (im.ri && s.nint != im.nint_cap) stat |= JPEGQS_DECODE_RESTART;
		if (s.nint > im.nint_cap) s.nint = im.nint_cap;
		s.unst.resize(s.unst.size() + 8, 0);
	}
	/* first scans: subsequences, chain, placement, final decode */
	for (size_t j = 0; j < plan.size(); j++) {
		const QsSeg &sg = plan[j].seg;
		const QdImg &im = sg.im;
		Seg &s = sd[j];
		if (!qs_first(sg.kind)) continue;
		std::vector<uint32_t> ivsub0(s.nint);
		uint32_t nsub = 0;
		for (uint32_t k = 0; k < s.nint; k++) {
			uint32_t b0 = s.ivstart[k], b1 = k + 1 < s.nint ? s.ivstart[k + 1] : s.nbytes;
			if (b1 < b0) { b1 = b0; stat |= JPEGQS_DECODE_RESTART; }
			uint32_t ns = (b1 - b0 + im.sub_bytes - 1) / im.sub_bytes;
			ivsub0[k] = nsub; nsub += ns ? ns : 1;
		}
		if (nsub > im.nsub_cap) { nsub = im.nsub_cap; stat |= JPEGQS_DECODE_UNITS; }
		std::vector<QdSub> sub(nsub);
		QsView v;
		qs_view(sg, s.tab.data(), s.unst.data(), s.nbytes, &v);
		auto span = [&](uint32_t q) { return qd_span(im, s.ivstart.data(), ivsub0.data(), s.nint, s.nbytes, nsub, q); };
		for (uint32_t q = 0; q < nsub; q++) {                     /* qs_sync mode 0: speculative decodes */
			QdSpan sp = span(q);
			QsView w = v; w.rd.lim = (uint32_t)(sp.iv_end >> 3);
			QdSub me = {};
			qs_path(w, sp.begin << 4, sp.end, sp.iv_end, sp.last, NULL, &me);
			me.iv = sp.iv; me.sync_units = 0;
			sub[q] = me;
		}
		/* qs_chain (the synchronisation rounds only shorten it: its fixed point is the same) */
		for (uint32_t q = 1; q < nsub; q++)
			if (sub[q].iv == sub[q - 1].iv && sub[q].entry != sub[q - 1].exit) {
				QdSpan sp = span(q);
				QsView w = v; w.rd.lim = (uint32_t)(sp.iv_end >> 3);
				QdSub old = sub[q], nw = old;
				nw.sync_units += qs_path(w, sub[q - 1].exit, sp.end, sp.iv_end, sp.last, &old, &nw);
				sub[q] = nw;
			}
		/* qs_place */
		uint64_t g = 0, tot = (uint64_t)im.nmcu * im.nblk; int32_t pred[4] = { 0, 0, 0, 0 };
		for (uint32_t q = 0; q < nsub; q++) {
			QdSpan sp = span(q);
			QdSub &sb = sub[q];
			if (sp.first) { g = 0; for (int c = 0; c < 4; c++) pred[c] = 0; }
			sb.g0 = (uint32_t)(g > tot ? tot : g);
			for (int c = 0; c < 4; c++) sb.pred[c] = pred[c];
			for (uint32_t r = 0; r < im.nblk; r++) pred[im.u_comp[(g + r) % im.nblk]] += sb.dcs[r];
			stat |= qs_place_check(sg, sb, sp, g, tot, s.nint);
			g += sb.cnt;
		}
		if (nsub < s.nint) stat |= JPEGQS_DECODE_UNITS;
		/* qs_final */
		for (uint32_t q = 0; q < nsub; q++) {
			QsView w = v;
			uint32_t iv = sub[q].iv;
			w.rd.lim = iv + 1 < s.nint ? s.ivstart[iv + 1] : s.nbytes;
			for (uint32_t k = 0; k < im.nblk; k++) { w.dc[k] = s.tab.data() + im.u_dc[k]; w.ac[k] = s.tab.data() + 4 + im.u_ac[k]; }
			w.period = im.nblk;
			stat |= qs_final_sub(sg, w, sub[q], s.nint);
		}
	}
	/* DC refinement scans */
	for (size_t j = 0; j < plan.size(); j++) {
		const QsSeg &sg = plan[j].seg;
		if (sg.kind != QS_DCR) continue;
		for (uint64_t u = 0; u < (uint64_t)sg.im.nmcu * sg.im.nblk; u++) {
			int16_t *dst; bool one;
			stat |= qs_dcr_unit(sg, sd[j].unst.data(), sd[j].ivstart.data(), sd[j].nint, sd[j].nbytes, u, &dst, &one);
			if (dst && one) dst[0] = (int16_t)(dst[0] | (1 << sg.Al));
		}
	}
	/* AC refinement scans, level after level */
	uint32_t maxlevel = 0;
	for (const QsPlan &pl : plan) if (pl.seg.kind == QS_ACR) maxlevel = std::max(maxlevel, pl.seg.level);
	for (uint32_t lv = 0; lv <= maxlevel; lv++)
		for (size_t j = 0; j < plan.size(); j++) {
			const QsSeg &sg = plan[j].seg;
			const Seg &s = sd[j];
			if (sg.kind != QS_ACR || sg.level != lv) continue;
			for (uint32_t k = 0; k < s.nint; k++) {
				uint32_t b0 = s.ivstart[k], b1 = k + 1 < s.nint ? s.ivstart[k + 1] : s.nbytes;
				if (b1 < b0) b1 = b0;
				stat |= qs_acr_interval(sg, s.tab.data() + 4 + sg.im.u_ac[0], s.unst.data(), b0, b1, (uint64_t)k * sg.im.ri,
						(uint64_t)qd_expect(sg.im, k, s.nint), zz);
			}
		}
	*status = (int32_t)stat;
	return 0;
}
