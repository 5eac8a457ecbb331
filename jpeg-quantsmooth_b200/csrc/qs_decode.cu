/*
 * qs_decode.cu - jpegqs_cuda_decode_async: the entropy-coded data of sequential Huffman JPEG files
 * decoded to quantized coefficients on the GPU, and jpegqs_cuda_decode_model, the same steps on the
 * CPU.  DESIGN.md section 3.6 describes the scheme; in short:
 *
 *   unit      one block: a DC code with its value bits, then AC codes up to EOB or coefficient 63.
 *   period P  the smallest period of the MCU's (DC table, AC table) sequence.  A decoder state is
 *             (bit position, unit index mod P): for one table pair (CMYK, untransformed RGB) that is
 *             a block boundary, for 4:2:0 YCbCr the MCU.
 *   bytes     FF00 removed, RSTn found and checked, the segment's end found (qd_scan / qd_seg /
 *             qd_compact: memory-bound passes over the data).
 *   subs      every restart interval (the whole segment without restart markers) is cut into
 *             subsequences of key-9 bytes.  Each is decoded speculatively from its first bit with
 *             phase 0 (qd_sync, mode 0), then the states are synchronised: rounds inside a thread
 *             block until nothing changes, one more grid-wide round (mode 1), then qd_chain walks
 *             every image in order and re-decodes any subsequence whose entry is not its
 *             predecessor's exit.  Re-decoding runs beside the old decode and stops where the two
 *             meet (same position, same phase): from there on they are the same.
 *   place     a segmented scan of the unit counts (reset at every restart) gives each subsequence's
 *             first unit, and one of the DC differences its predictors (qd_place).
 *   decode    each subsequence decodes its units once more, from its proven entry, into the arrays
 *             (qd_final), and checks that it ends where the next one starts.
 * Every MCU is decoded in the final pass from a state the chain of decodes from a true start (the
 * segment start or a restart marker) reached, so the result is the sequential decoder's.
 */
#include <stdio.h>
#include <memory>
#include <vector>
#include "qs_decode.h"

/* ---------------------------------------------------------------- paths: decodes from a state */
struct QdView {                        /* what a path needs of an image */
	const QdHuff *dc[QD_MAX_UNITS], *ac[QD_MAX_UNITS];   /* by phase */
	uint32_t period, nblk;
	QdRd rd;
};
HD static inline void qd_view(const QdImg &im, const QdHuff *tab, const uint8_t *unst, uint32_t lim, QdView *v) {
	for (uint32_t p = 0; p < im.period; p++) { v->dc[p] = tab + im.u_dc[p]; v->ac[p] = tab + 4 + im.u_ac[p]; }
	v->period = im.period; v->nblk = im.nblk; v->rd.d = unst; v->rd.lim = lim;
}


/* Decodes from state `start` until a unit start at or past end_bits (or the padding before the
 * interval end when last), into *out.  With old (a decode of the same subsequence from another
 * entry), it runs beside that decode and stops where the two meet; the rest is taken from old.
 * Returns the units decoded from `start`. */
HD static uint32_t qd_path(const QdView &v, uint64_t start, uint64_t end_bits, uint64_t iv_end, bool last,
		const QdSub *old, QdSub *out) {
	uint64_t a = start >> 4, b = 0; uint32_t pa = (uint32_t)(start & 15), pb = 0, ca = 0, cb = 0, ra = 0, rb = 0, n = 0;
	int32_t da[QD_MAX_UNITS], db[QD_MAX_UNITS];
	uint64_t ea = 0;
	bool hasb = old && old->entry != QD_NONE;
	for (int i = 0; i < QD_MAX_UNITS; i++) da[i] = db[i] = 0;
	if (hasb) { b = old->entry >> 4; pb = (uint32_t)(old->entry & 15); }
	for (;;) {
		if (hasb && a == b && pa == pb) {                /* met the old decode: the rest is its */
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
		if (!hasb || cb >= old->cnt || a <= b) {
			uint32_t e = 0; int diff;
			uint64_t na = qd_unit(v.rd, a, v.dc[pa], v.ac[pa], &diff, NULL, &e);
			if (e) ea = a << 8 | e;
			da[ra] += diff; ra = ra + 1 == v.nblk ? 0 : ra + 1;
			a = na; pa = pa + 1 == v.period ? 0 : pa + 1; ca++; n++;
		} else {
			uint32_t e = 0; int diff;
			uint64_t nb = qd_unit(v.rd, b, v.dc[pb], v.ac[pb], &diff, NULL, &e);
			db[rb] += diff; rb = rb + 1 == v.nblk ? 0 : rb + 1;
			b = nb; pb = pb + 1 == v.period ? 0 : pb + 1; cb++;
		}
	}
	out->entry = start;
	return n;
}

/* the final decode of subsequence s (entry, cnt, g0 and pred placed) into the arrays */
HD static inline uint32_t qd_final_sub(const QdImg &im, const QdView &v, const QdSub &sb) {
	uint32_t err = 0;
	if (sb.entry == QD_NONE) return 0;
	uint64_t pos = sb.entry >> 4;
	int32_t pred[4] = { sb.pred[0], sb.pred[1], sb.pred[2], sb.pred[3] };
	uint64_t u = (uint64_t)sb.iv * im.ri * im.nblk + sb.g0;
	uint32_t k = (uint32_t)(u % im.nblk); uint64_t m = u / im.nblk;
	for (uint32_t i = 0; i < sb.cnt; i++) {
		int16_t blk[64];
		for (int j = 0; j < 64; j++) blk[j] = 0;
		int diff; uint32_t c = im.u_comp[k];
		pos = qd_unit(v.rd, pos, v.dc[k % v.period], v.ac[k % v.period], &diff, blk, &err);
		pred[c] += diff;
		blk[0] = (int16_t)pred[c];
		if (m < im.nmcu) {
			uint64_t bx = (uint64_t)(m % im.nx) * im.u_hs[k] + im.u_h[k], by = (uint64_t)(m / im.nx) * im.u_vs[k] + im.u_v[k];
			uint32_t fc = im.u_comp[k];
			if (bx < im.wblk[fc] && by < im.hblk[fc]) {
				int16_t *dst = im.coef[fc] + ((size_t)by * im.wblk[fc] + bx) * 64;
#ifdef __CUDA_ARCH__
				for (int j = 0; j < 8; j++) reinterpret_cast<int4 *>(dst)[j] = reinterpret_cast<const int4 *>(blk)[j];
#else
				memcpy(dst, blk, sizeof(blk));
#endif
			}
		} else err |= JPEGQS_DECODE_UNITS;
		if (++k == im.nblk) { k = 0; m++; }
	}
	if (pos != sb.exit >> 4) err |= JPEGQS_DECODE_UNITS;
	return err;
}

/* ---------------------------------------------------------------- kernels */
struct QdSetupPack {
	QdImg img[QD_PACK];
	uint8_t bits[QD_PACK][8][17];
	uint8_t val[QD_PACK][8][256];
	int n;
};
static_assert(sizeof(QdSetupPack) <= 32000, "QdSetupPack exceeds the kernel parameter space");

/* blockIdx.x = table 0..7, blockIdx.y = image: derived tables, descriptor, state, status */
__global__ void qd_setup_kernel(const __grid_constant__ QdSetupPack p) {
	int i = blockIdx.y, t = blockIdx.x;
	if (i >= p.n) return;
	const QdImg &im = p.img[i];
	if (threadIdx.x == 0) {
		if (p.bits[i][t][0] == 1) qd_build(im.tab + t, p.bits[i][t], p.val[i][t]);   /* bits[0] = 1: present */
		if (t == 0) {
			*reinterpret_cast<QdImg *>(reinterpret_cast<char *>(im.tab) - 2048) = im;
			memset(im.st, 0, sizeof(QdState));
			*im.status = 0;
		}
	}
}

struct QdPtrs { const QdImg *img[QD_PACK]; int n; };

__global__ void __launch_bounds__(QD_BT) qd_scan_kernel(const __grid_constant__ QdPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	qd_scan_body(*P.img[blockIdx.y], blockIdx.x);
}

__global__ void __launch_bounds__(QD_SCAN_T) qd_seg_kernel(const __grid_constant__ QdPtrs P) {
	if ((int)blockIdx.x >= P.n) return;
	qd_seg_body(*P.img[blockIdx.x]);
}

__global__ void __launch_bounds__(QD_BT) qd_compact_kernel(const __grid_constant__ QdPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	qd_compact_body(*P.img[blockIdx.y], blockIdx.x);
}

__global__ void __launch_bounds__(QD_SCAN_T) qd_iv_kernel(const __grid_constant__ QdPtrs P) {
	if ((int)blockIdx.x >= P.n) return;
	qd_iv_body(*P.img[blockIdx.x]);
}

/* mode 0: speculative decode of every subsequence, then rounds inside the block; mode 1: one more
 * round in which a block's first subsequence also takes its predecessor's exit from memory */
__global__ void __launch_bounds__(QD_ST) qd_sync_kernel(const __grid_constant__ QdPtrs P, int mode) {
	if ((int)blockIdx.y >= P.n) return;
	const QdImg &im = *P.img[blockIdx.y];
	const QdState *st = im.st;
	uint32_t nsub = st->nsub, s = blockIdx.x * QD_ST + threadIdx.x;
	if (blockIdx.x * QD_ST >= nsub) return;
	__shared__ uint64_t s_exit[QD_ST];
	QdView v;
	qd_view(im, im.tab, im.unst, st->nbytes, &v);
	bool act = s < nsub;
	QdSpan sp = {};
	QdSub me = {};
	me.entry = QD_NONE;
	if (act) {
		sp = qd_span(im, im.ivstart, im.ivsub0, st->nint, st->nbytes, nsub, s);
		v.rd.lim = (uint32_t)(sp.iv_end >> 3);
		if (mode == 0) {
			qd_path(v, sp.begin << 4, sp.end, sp.iv_end, sp.last, NULL, &me);
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
			/* The previous thread block of this launch may be rewriting that record right now: the
			 * read sees its exit before or after the rewrite (one aligned 64-bit load, never torn),
			 * and either is a state some decode reached.  A stale value only costs a re-decode;
			 * qd_chain then checks every entry against the final exits in order, so the fixed
			 * point does not depend on which one was read.  (The CPU model reads a snapshot.) */
			else if (mode == 1) want = *(volatile const uint64_t *)&im.sub[s - 1].exit;
			else want = me.entry;
			if (want != me.entry) {
				QdSub nw = me;
				nw.sync_units += qd_path(v, want, sp.end, sp.iv_end, sp.last, &me, &nw);
				me = nw; changed = true;
			}
		}
		if (!__syncthreads_or(changed)) break;
		mode = mode == 1 ? 2 : mode;                     /* the memory read happens once */
	}
	if (act) im.sub[s] = me;
}

/* per image, one warp: in order, every subsequence whose entry is not its predecessor's exit is
 * decoded again from that exit - the fixed point the rounds nearly always reached already */
__global__ void __launch_bounds__(32) qd_chain_kernel(const __grid_constant__ QdPtrs P) {
	if ((int)blockIdx.x >= P.n) return;
	const QdImg &im = *P.img[blockIdx.x];
	const QdState *st = im.st;
	uint32_t nsub = st->nsub, lane = threadIdx.x;
	QdView v;
	qd_view(im, im.tab, im.unst, st->nbytes, &v);
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
			QdView w = v;
			w.rd.lim = (uint32_t)(sp.iv_end >> 3);
			QdSub old = im.sub[f], nw = old;
			nw.sync_units += qd_path(w, im.sub[f - 1].exit, sp.end, sp.iv_end, sp.last, &old, &nw);
			im.sub[f] = nw;
			__threadfence_block();
		}
		__syncwarp();
		base = f + 1;
	}
}

/* per image: segmented scans (reset at every restart interval) of the unit counts and the DC
 * differences; unit-count, restart-end and path-error checks */
struct QdAcc { uint32_t flag, cnt; };
struct QdDc { uint32_t flag; int32_t v[4]; };
__global__ void __launch_bounds__(QD_SCAN_T) qd_place_kernel(const __grid_constant__ QdPtrs P) {
	if ((int)blockIdx.x >= P.n) return;
	const QdImg &im = *P.img[blockIdx.x];
	const QdState *st = im.st;
	typedef cub::BlockScan<QdAcc, QD_SCAN_T> S1;
	typedef cub::BlockScan<QdDc, QD_SCAN_T> S2;
	__shared__ union { typename S1::TempStorage a; typename S2::TempStorage b; } tmp;
	struct Op1 { __device__ QdAcc operator()(QdAcc a, QdAcc b) const { return b.flag ? b : QdAcc{ a.flag, a.cnt + b.cnt }; } };
	struct Op2 { __device__ QdDc operator()(QdDc a, QdDc b) const {
		if (b.flag) return b;
		QdDc r; r.flag = a.flag; for (int c = 0; c < 4; c++) r.v[c] = a.v[c] + b.v[c]; return r; } };
	uint32_t nsub = st->nsub, nint = st->nint;
	QdAcc c1 = { 1, 0 };
	QdDc c2 = { 1, { 0, 0, 0, 0 } };
	uint32_t bad = 0;
	for (uint32_t base = 0; base < nsub; base += QD_SCAN_T) {
		uint32_t s = base + threadIdx.x;
		bool act = s < nsub;
		QdSub sb = {};
		QdSpan sp = {};
		if (act) { sb = im.sub[s]; sp = qd_span(im, im.ivstart, im.ivsub0, nint, st->nbytes, nsub, s); }
		QdAcc a = { act && sp.first ? 1u : 0u, act ? sb.cnt : 0u }, ae, aagg;
		S1(tmp.a).ExclusiveScan(a, ae, c1, Op1(), aagg);
		__syncthreads();
		uint32_t g0 = ae.cnt;
		if (a.flag) g0 = 0;
		/* the DC sums per frame component: unit g0 + r of the interval is unit (g0 + r) mod nblk of its MCU */
		QdDc d = { a.flag, { 0, 0, 0, 0 } };
		if (act) for (uint32_t r = 0; r < im.nblk; r++) d.v[im.u_comp[(g0 + r) % im.nblk]] += sb.dcs[r];
		QdDc de, dagg;
		S2(tmp.b).ExclusiveScan(d, de, c2, Op2(), dagg);
		__syncthreads();
		if (act) {
			QdSub &w = im.sub[s];
			w.g0 = g0;
			for (int c = 0; c < 4; c++) w.pred[c] = d.flag ? 0 : de.v[c];
			if (sb.entry == QD_NONE) bad |= JPEGQS_DECODE_UNITS;
			if (sb.err) bad |= (uint32_t)(sb.err & 0xFF);
			if (sb.entry != QD_NONE && (uint32_t)(sb.entry & 15) != g0 % im.period) bad |= JPEGQS_DECODE_UNITS;
			if (sp.last) {
				if ((int64_t)g0 + sb.cnt != qd_expect(im, sp.iv, nint)) bad |= JPEGQS_DECODE_UNITS;
				uint64_t x = sb.exit >> 4;
				if (x > sp.iv_end) bad |= JPEGQS_DECODE_TRUNCATED;
			}
		}
		c1 = Op1()(c1, aagg);
		c2 = Op2()(c2, dagg);
		__syncthreads();
	}
	if (nsub < nint) bad |= JPEGQS_DECODE_UNITS;
	if (bad) atomicOr(im.status, (int)bad);
}

__global__ void __launch_bounds__(QD_ST) qd_final_kernel(const __grid_constant__ QdPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QdImg &im = *P.img[blockIdx.y];
	const QdState *st = im.st;
	uint32_t s = blockIdx.x * QD_ST + threadIdx.x;
	if (s >= st->nsub) return;
	QdView v;
	qd_view(im, im.tab, im.unst, st->nbytes, &v);
	QdSub sb = im.sub[s];
	uint32_t nint = st->nint;
	uint32_t ivend = sb.iv + 1 < nint ? im.ivstart[sb.iv + 1] : st->nbytes;
	v.rd.lim = ivend;
	/* the final decode maps units by their index mod nblk: the tables of unit k of the MCU */
	for (uint32_t k = 0; k < im.nblk && k < QD_MAX_UNITS; k++) { v.dc[k] = im.tab + im.u_dc[k]; v.ac[k] = im.tab + 4 + im.u_ac[k]; }
	v.period = im.nblk;
	uint32_t e = qd_final_sub(im, v, sb);
	if (e) atomicOr(im.status, (int)e);
}

/* ---------------------------------------------------------------- host: checks, workspace, launches */
struct jpegqs_cuda_ctx;
void qs_ctx_decode_info(jpegqs_cuda_ctx *ctx, int *device, cudaStream_t *stream, int *sub_bytes);
void qs_ctx_decode_done(jpegqs_cuda_ctx *ctx, int launches, const char *err);
extern "C" void qs_set_host_error(const char *msg);

static size_t qd_a256(size_t x) { return (x + 255) & ~(size_t)255; }

struct QdPlan {                        /* one image, host side */
	QdImg img;
	uint8_t bits[8][17], val[8][256];
	size_t bytes, nsub_grid;
};

static bool qd_same_table(const jpegqs_cuda_scan *s, int dc, int a, int b) {
	const uint8_t *ba = dc ? s->dc_bits[a] : s->ac_bits[a], *bb = dc ? s->dc_bits[b] : s->ac_bits[b];
	const uint8_t *va = dc ? s->dc_val[a] : s->ac_val[a], *vb = dc ? s->dc_val[b] : s->ac_val[b];
	int n = 0;
	for (int l = 1; l <= 16; l++) { if (ba[l] != bb[l]) return false; n += ba[l]; }
	return !memcmp(va, vb, n > 256 ? 256 : n);
}

/* checks image i and fills its plan (pointers only when ptrs); returns 0 or a message */
static const char *qd_check(const jpegqs_cuda_image *im, const jpegqs_cuda_scan *sc, size_t len, bool ptrs,
		int sub_bytes, QdPlan *pl) {
	memset(pl, 0, sizeof(*pl));
	QdImg &d = pl->img;
	int nc = im->ncomp;
	if (nc < 1 || nc > 4 || sc->ncomp != nc) return "ncomp outside 1..4 or unequal to the scan's";
	if (sc->entropy_offset >= len) return "entropy_offset at or beyond data_len";
	if (len - sc->entropy_offset > 0xFFFFFFF0ull) return "entropy-coded data longer than 4 GB";
	if (sc->restart_interval > 65535) return "restart interval beyond 65535";
	int seen = 0, maxh = 1, maxv = 1;
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
		d.wblk[c] = cc.wblk; d.hblk[c] = cc.hblk; d.coef[c] = cc.coef;
	}
	for (int k = 0; k < nc; k++) {
		int c = sc->comp[k];
		if (c < 0 || c >= nc || (seen >> c & 1)) return "scan components are not a permutation of the frame's";
		seen |= 1 << c;
		int td = sc->dc_tbl[k], ta = sc->ac_tbl[k];
		if (td < 0 || td > 3 || ta < 0 || ta > 3 || !sc->dc_present[td] || !sc->ac_present[ta]) return "a selector names an absent table";
	}
	/* tables: the ones the scan selects, checked as libjpeg does */
	for (int t = 0; t < 8; t++) {
		int dc = t < 4, j = t & 3, used = 0;
		for (int k = 0; k < nc; k++) used |= dc ? sc->dc_tbl[k] == j : sc->ac_tbl[k] == j;
		if (!used) continue;
		memcpy(pl->bits[t], dc ? sc->dc_bits[j] : sc->ac_bits[j], 17);
		memcpy(pl->val[t], dc ? sc->dc_val[j] : sc->ac_val[j], 256);
		pl->bits[t][0] = 1;
		QdHuff h;
		if (qd_build(&h, pl->bits[t], pl->val[t])) return "a selected Huffman table is invalid";
		if (dc) { int n = 0; for (int l = 1; l <= 16; l++) n += pl->bits[t][l]; for (int i = 0; i < n; i++) if (pl->val[t][i] > 15) return "a DC table holds a symbol > 15"; }
	}
	/* the units of one MCU (A.2.3; one component: not interleaved, one block) */
	uint32_t nb = 0;
	if (nc == 1) {
		d.nx = d.wblk[0]; d.ny = d.hblk[0];
		d.u_comp[0] = (uint8_t)sc->comp[0]; d.u_hs[0] = d.u_vs[0] = 1; d.u_h[0] = d.u_v[0] = 0;
		d.u_dc[0] = (uint8_t)sc->dc_tbl[0]; d.u_ac[0] = (uint8_t)sc->ac_tbl[0];
		nb = 1;
	} else {
		d.nx = (uint32_t)(((uint64_t)im->image_width + 8 * maxh - 1) / (8 * maxh));
		d.ny = (uint32_t)(((uint64_t)im->image_height + 8 * maxv - 1) / (8 * maxv));
		for (int k = 0; k < nc; k++) {
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
	/* the smallest period of the units' table sequence */
	for (d.period = 1; d.period < nb; d.period++) {
		if (nb % d.period) continue;
		uint32_t k;
		for (k = d.period; k < nb; k++)
			if (!qd_same_table(sc, 1, d.u_dc[k], d.u_dc[k - d.period]) || !qd_same_table(sc, 0, d.u_ac[k], d.u_ac[k - d.period])) break;
		if (k == nb) break;
	}
	d.ri = sc->restart_interval;
	d.nint_cap = d.ri ? (uint32_t)((nmcu + d.ri - 1) / d.ri) : 1;
	if (!d.nint_cap) d.nint_cap = 1;
	uint64_t L = len - sc->entropy_offset;
	d.off = sc->entropy_offset; d.len = len;
	d.nchunk = (uint32_t)((L + QD_CHUNK - 1) / QD_CHUNK);
	d.sub_bytes = (uint32_t)sub_bytes;
	d.nsub_cap = (uint32_t)(L / QD_SUB_MIN + d.nint_cap);
	pl->nsub_grid = L / (uint64_t)sub_bytes + d.nint_cap;
	pl->bytes = QD_FIXED + qd_a256(L + 8) + qd_a256(24 * (size_t)d.nchunk) + 2 * qd_a256(4 * (size_t)d.nint_cap) +
		qd_a256(96 * (size_t)d.nsub_cap);
	return NULL;
}

static void qd_carve(QdPlan *pl, char *w, int32_t *status) {
	QdImg &d = pl->img;
	uint64_t L = d.len - d.off;
	d.st = reinterpret_cast<QdState *>(w + 1024);
	d.tab = reinterpret_cast<QdHuff *>(w + 2048);
	w += QD_FIXED;
	d.unst = reinterpret_cast<uint8_t *>(w); w += qd_a256(L + 8);
	d.chunk = reinterpret_cast<QdChunk *>(w); w += qd_a256(24 * (size_t)d.nchunk);
	d.ivstart = reinterpret_cast<uint32_t *>(w); w += qd_a256(4 * (size_t)d.nint_cap);
	d.ivsub0 = reinterpret_cast<uint32_t *>(w); w += qd_a256(4 * (size_t)d.nint_cap);
	d.sub = reinterpret_cast<QdSub *>(w);
	d.status = status;
}

extern "C" int jpegqs_cuda_decode_workspace_bytes(int n, const jpegqs_cuda_image *imgs, const jpegqs_cuda_scan *scans,
		const size_t *data_len, size_t *bytes) {
	if (n < 0 || !bytes || (n && (!imgs || !scans || !data_len))) { qs_set_host_error("jpegqs_cuda_decode_workspace_bytes: NULL argument"); return JPEGQS_ERR_ARG; }
	size_t total = 0;
	for (int i = 0; i < n; i++) {
		QdPlan pl;
		const char *e = qd_check(&imgs[i], &scans[i], data_len[i], false, QD_SUB_MIN, &pl);
		if (e) { char m[256]; snprintf(m, sizeof(m), "jpegqs_cuda_decode_workspace_bytes: image %d: %s", i, e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
		total += pl.bytes;
	}
	*bytes = total;
	return 0;
}

#define QD_CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	snprintf(msg, sizeof(msg), "%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
	qs_ctx_decode_done(ctx, launches, msg); return JPEGQS_ERR_CUDA; } } while (0)

extern "C" int jpegqs_cuda_decode_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_scan *scans, const uint8_t *const *data_dev, const size_t *data_len,
		void *workspace, size_t workspace_bytes, int32_t *status_dev, void *stream) {
	char msg[512] = "";
	int launches = 0;
	if (!ctx) return JPEGQS_ERR_ARG;
	int device, sub_bytes; cudaStream_t st;
	qs_ctx_decode_info(ctx, &device, &st, &sub_bytes);
	if (stream) st = (cudaStream_t)stream;
	if (n < 0 || (n && (!imgs || !scans || !data_dev || !data_len || !status_dev || !workspace))) {
		qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_decode_async: NULL argument"); return JPEGQS_ERR_ARG;
	}
	if ((uintptr_t)workspace & 255) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_decode_async: workspace not 256-byte aligned"); return JPEGQS_ERR_ARG; }
	std::vector<QdPlan> plan((size_t)n);
	size_t need = 0;
	for (int i = 0; i < n; i++) {
		const char *e = data_dev[i] ? qd_check(&imgs[i], &scans[i], data_len[i], true, sub_bytes, &plan[i]) : "data_dev entry NULL";
		if (e) { snprintf(msg, sizeof(msg), "jpegqs_cuda_decode_async: image %d: %s", i, e); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
		plan[i].img.data = data_dev[i];
		need += plan[i].bytes;
	}
	if (workspace_bytes < need) {
		snprintf(msg, sizeof(msg), "jpegqs_cuda_decode_async: workspace of %zu bytes, %zu needed", workspace_bytes, need);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (!n) { qs_ctx_decode_done(ctx, 0, ""); return 0; }
	QD_CK(cudaSetDevice(device));
	char *w = (char *)workspace;
	for (int i = 0; i < n; i++) { qd_carve(&plan[i], w, status_dev + i); w += plan[i].bytes; }
	for (int g0 = 0; g0 < n; g0 += QD_PACK) {
		int g = n - g0 < QD_PACK ? n - g0 : QD_PACK;
		std::unique_ptr<QdSetupPack> hold(new QdSetupPack());   /* per call (20 KB: not on the stack) */
		QdSetupPack &pack = *hold;
		QdPtrs P;
		memset(&pack, 0, sizeof(pack)); memset(&P, 0, sizeof(P));
		pack.n = g; P.n = g;
		uint32_t maxchunk = 1; size_t maxsub = 1;
		for (int j = 0; j < g; j++) {
			const QdPlan &pl = plan[g0 + j];
			pack.img[j] = pl.img;
			memcpy(pack.bits[j], pl.bits, sizeof(pl.bits)); memcpy(pack.val[j], pl.val, sizeof(pl.val));
			P.img[j] = reinterpret_cast<const QdImg *>(reinterpret_cast<const char *>(pl.img.tab) - 2048);
			if (pl.img.nchunk > maxchunk) maxchunk = pl.img.nchunk;
			if (pl.nsub_grid > maxsub) maxsub = pl.nsub_grid;
		}
		uint32_t subblocks = (uint32_t)((maxsub + QD_ST - 1) / QD_ST);
		qd_setup_kernel<<<dim3(8, g), 32, 0, st>>>(pack); launches++;
		qd_scan_kernel<<<dim3(maxchunk, g), QD_BT, 0, st>>>(P); launches++;
		qd_seg_kernel<<<g, QD_SCAN_T, 0, st>>>(P); launches++;
		qd_compact_kernel<<<dim3(maxchunk, g), QD_BT, 0, st>>>(P); launches++;
		qd_iv_kernel<<<g, QD_SCAN_T, 0, st>>>(P); launches++;
		qd_sync_kernel<<<dim3(subblocks, g), QD_ST, 0, st>>>(P, 0); launches++;
		qd_sync_kernel<<<dim3(subblocks, g), QD_ST, 0, st>>>(P, 1); launches++;
		qd_chain_kernel<<<g, 32, 0, st>>>(P); launches++;
		qd_place_kernel<<<g, QD_SCAN_T, 0, st>>>(P); launches++;
		qd_final_kernel<<<dim3(subblocks, g), QD_ST, 0, st>>>(P); launches++;
		QD_CK(cudaGetLastError());
	}
	qs_ctx_decode_done(ctx, launches, "");
	return 0;
}

/* ---------------------------------------------------------------- the CPU model */
extern "C" int jpegqs_cuda_decode_model(const jpegqs_cuda_image *img, const jpegqs_cuda_scan *scan, const uint8_t *data,
		size_t data_len, int sub_bytes, int32_t *status, uint32_t *overrun, size_t overrun_cap, size_t *nsub_out) {
	if (!img || !scan || !data || !status) { qs_set_host_error("jpegqs_cuda_decode_model: NULL argument"); return JPEGQS_ERR_ARG; }
	if (sub_bytes < QD_SUB_MIN) { qs_set_host_error("jpegqs_cuda_decode_model: sub_bytes below 32"); return JPEGQS_ERR_ARG; }
	QdPlan pl;
	const char *e = qd_check(img, scan, data_len, true, sub_bytes, &pl);
	if (e) { char m[256]; snprintf(m, sizeof(m), "jpegqs_cuda_decode_model: %s", e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
	QdImg &im = pl.img;
	im.data = data;
	uint32_t stat = 0;
	std::vector<QdHuff> tab(8);
	for (int t = 0; t < 8; t++) if (pl.bits[t][0] == 1) qd_build(&tab[t], pl.bits[t], pl.val[t]);
	/* byte passes */
	std::vector<uint8_t> unst;
	std::vector<uint32_t> ivstart(im.nint_cap, 0);
	uint32_t nrst = 0;
	{
		bool ri = im.ri != 0;
		for (uint64_t p = im.off; p < im.len; p++) {
			bool t, k, r;
			qd_byte_class(data, im.off, im.len, p, ri, &t, &k, &r);
			if (t) break;
			if (r) {
				if ((uint32_t)(data[p + 1] & 7) != (nrst & 7)) stat |= JPEGQS_DECODE_RESTART;
				if (nrst + 1 < im.nint_cap) ivstart[nrst + 1] = (uint32_t)unst.size();
				nrst++;
			}
			if (k) unst.push_back(data[p]);
		}
	}
	uint32_t nbytes = (uint32_t)unst.size();
	uint32_t nint = im.ri ? nrst + 1 : 1;
	if (im.ri && nint != im.nint_cap) stat |= JPEGQS_DECODE_RESTART;
	if (nint > im.nint_cap) nint = im.nint_cap;
	unst.resize(unst.size() + 8, 0);
	std::vector<uint32_t> ivsub0(nint);
	uint32_t nsub = 0;
	for (uint32_t k = 0; k < nint; k++) {
		uint32_t b0 = ivstart[k], b1 = k + 1 < nint ? ivstart[k + 1] : nbytes;
		if (b1 < b0) { b1 = b0; stat |= JPEGQS_DECODE_RESTART; }
		uint32_t ns = (b1 - b0 + im.sub_bytes - 1) / im.sub_bytes;
		ivsub0[k] = nsub; nsub += ns ? ns : 1;
	}
	if (nsub > im.nsub_cap) { nsub = im.nsub_cap; stat |= JPEGQS_DECODE_UNITS; }
	std::vector<QdSub> sub(nsub);
	QdView v;
	qd_view(im, tab.data(), unst.data(), nbytes, &v);
	auto span = [&](uint32_t s) { return qd_span(im, ivstart.data(), ivsub0.data(), nint, nbytes, nsub, s); };
	auto redo = [&](uint32_t s, uint64_t want) {
		QdSpan sp = span(s);
		QdView w = v; w.rd.lim = (uint32_t)(sp.iv_end >> 3);
		QdSub old = sub[s], nw = old;
		nw.sync_units += qd_path(w, want, sp.end, sp.iv_end, sp.last, &old, &nw);
		sub[s] = nw;
	};
	/* qd_sync mode 0: speculative decodes, then rounds inside blocks of QD_ST */
	for (uint32_t s = 0; s < nsub; s++) {
		QdSpan sp = span(s);
		QdView w = v; w.rd.lim = (uint32_t)(sp.iv_end >> 3);
		QdSub me = {};
		qd_path(w, sp.begin << 4, sp.end, sp.iv_end, sp.last, NULL, &me);
		me.iv = sp.iv; me.sync_units = 0;
		sub[s] = me;
	}
	for (int mode = 0; mode < 2; mode++) {
		std::vector<uint64_t> snap(nsub);
		for (uint32_t s = 0; s < nsub; s++) snap[s] = sub[s].exit;
		for (uint32_t b0 = 0; b0 < nsub; b0 += QD_ST) {
			uint32_t b1 = b0 + QD_ST < nsub ? b0 + QD_ST : nsub;
			bool first_round = true;
			for (;;) {
				std::vector<uint64_t> ex(b1 - b0);
				for (uint32_t s = b0; s < b1; s++) ex[s - b0] = sub[s].exit;
				bool changed = false;
				for (uint32_t s = b0; s < b1; s++) {
					if (span(s).first) continue;
					uint64_t want;
					if (s > b0) want = ex[s - b0 - 1];
					else if (mode == 1 && first_round) want = snap[s - 1];
					else want = sub[s].entry;
					if (want != sub[s].entry) { redo(s, want); changed = true; }
				}
				first_round = false;
				if (!changed) break;
			}
		}
	}
	/* qd_chain */
	for (uint32_t s = 1; s < nsub; s++)
		if (sub[s].iv == sub[s - 1].iv && sub[s].entry != sub[s - 1].exit) redo(s, sub[s - 1].exit);
	/* qd_place */
	{
		uint32_t g = 0; int32_t pred[4] = { 0, 0, 0, 0 };
		for (uint32_t s = 0; s < nsub; s++) {
			QdSpan sp = span(s);
			QdSub &sb = sub[s];
			if (sp.first) { g = 0; for (int c = 0; c < 4; c++) pred[c] = 0; }
			sb.g0 = g;
			for (int c = 0; c < 4; c++) sb.pred[c] = pred[c];
			for (uint32_t r = 0; r < im.nblk; r++) pred[im.u_comp[(g + r) % im.nblk]] += sb.dcs[r];
			g += sb.cnt;
			if (sb.entry == QD_NONE) stat |= JPEGQS_DECODE_UNITS;
			if (sb.err) stat |= (uint32_t)(sb.err & 0xFF);
			if (sb.entry != QD_NONE && (uint32_t)(sb.entry & 15) != sb.g0 % im.period) stat |= JPEGQS_DECODE_UNITS;
			if (sp.last) {
				if ((int64_t)g != qd_expect(im, sp.iv, nint)) stat |= JPEGQS_DECODE_UNITS;
				if ((sb.exit >> 4) > sp.iv_end) stat |= JPEGQS_DECODE_TRUNCATED;
			}
		}
		if (nsub < nint) stat |= JPEGQS_DECODE_UNITS;
	}
	/* qd_final */
	for (uint32_t s = 0; s < nsub; s++) {
		QdView w = v;
		uint32_t iv = sub[s].iv;
		w.rd.lim = iv + 1 < nint ? ivstart[iv + 1] : nbytes;
		for (uint32_t k = 0; k < im.nblk; k++) { w.dc[k] = tab.data() + im.u_dc[k]; w.ac[k] = tab.data() + 4 + im.u_ac[k]; }
		w.period = im.nblk;
		stat |= qd_final_sub(im, w, sub[s]);
	}
	if (overrun)
		for (uint32_t s = 0; s < nsub && s < overrun_cap; s++)
			overrun[s] = s + 1 < nsub && sub[s + 1].iv == sub[s].iv ? sub[s + 1].sync_units : 0;
	if (nsub_out) *nsub_out = nsub;
	*status = (int32_t)stat;
	return 0;
}
