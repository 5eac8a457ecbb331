/*
 * qs_encode.cu - jpegqs_cuda_encode_async: quantized coefficients on the GPU written as the sequential
 * Huffman JPEG file the jpegqs tool's writer (jpegcoef.c jq_write) writes for them, and
 * jpegqs_cuda_encode_model, the same steps on the CPU.  DESIGN.md section 3.7 describes the scheme; in
 * short:
 *
 *   unit      one block of the single interleaved scan, in MCU order.  Blocks of the MCU padding (past
 *             wblk / hblk) code a DC difference of 0 and an EOB, as jq_write and libjpeg's jctrans.c do.
 *   predictor the DC of the last REAL block of the unit's component before it.  The real blocks of an
 *             MCU form a rectangle that always holds its first block, so the predictor follows from
 *             the unit's index alone: encoding has no serial dependency.
 *   count     with optimize, every unit adds its symbols to per-image histograms (qe_count), and one
 *             warp per table builds jq_write's optimal table from them (qe_table, T.81 K.2).
 *   length    every unit's bit length with the final tables (qe_len); a scan over tiles of units
 *             (qe_tscan) and one inside each tile give every unit its bit offset.
 *   emit      every unit writes its bits into a zeroed word buffer (qe_zero, qe_emit): words it owns
 *             alone by plain stores, the two it may share with its neighbours by atomicOr.
 *   stuff     0xFF bytes are counted per chunk (qe_ffcount), the counts scanned (qe_fscan, which also
 *             decides length, status and EOI), and the chunks copied with a 0x00 after each 0xFF
 *             (qe_copy).  The prefix and the DQT / SOF / DHT / SOS segments come from qe_table.
 */
#include <cuda_runtime.h>
#include <cub/block/block_scan.cuh>
#include <cub/block/block_reduce.cuh>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <memory>
#include <vector>
#include "../../include/jpegqs_cuda.h"

#define HD __host__ __device__
#define QE_T 256                       /* units per tile (threads of the unit passes)        */
#define QE_BT 256                      /* threads of the byte passes: 16 bytes each           */
#define QE_CHUNK (QE_BT * 16)          /* unstuffed bytes per chunk                           */
#define QE_SCAN_T 1024                 /* threads of the per-image scans                      */
#define QE_MAX_UNITS 10                /* blocks per MCU (libjpeg C_MAX_BLOCKS_IN_MCU)         */
#define QE_PACK 16                     /* images per launch group                             */
#define QE_FIXED 32768                 /* descriptor + state + four tables per image          */
#define QE_BLOCK_BITS 1665ull          /* 16 + 11 DC bits, 63 x (16 + 10) AC bits             */
#define QE_HEAD_MAX 1680ull            /* DQT, SOF, DHT, SOS, EOI at most                     */
#define QE_SENT 1000000000ull          /* ehuff_optimal's "no candidate" frequency            */

/* zig-zag -> natural order (T.81 figure A.6) and back */
__constant__ uint8_t qe_nat_dev[64] = {
	0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
	28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
	54, 47, 55, 62, 63 };
__constant__ uint8_t qe_zz_dev[64] = {
	0, 1, 5, 6, 14, 15, 27, 28, 2, 4, 7, 13, 16, 26, 29, 42, 3, 8, 12, 17, 25, 30, 41, 43, 9, 11, 18, 24, 31, 40, 44, 53,
	10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57,
	58, 62, 63 };
static const uint8_t qe_nat_host[64] = {
	0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
	28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
	54, 47, 55, 62, 63 };
static const uint8_t qe_zz_host[64] = {
	0, 1, 5, 6, 14, 15, 27, 28, 2, 4, 7, 13, 16, 26, 29, 42, 3, 8, 12, 17, 25, 30, 41, 43, 9, 11, 18, 24, 31, 40, 44, 53,
	10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57,
	58, 62, 63 };
HD static inline int qe_nat(int k) {
#ifdef __CUDA_ARCH__
	return qe_nat_dev[k];
#else
	return qe_nat_host[k];
#endif
}

/* T.81 K.3.3 example tables: BITS (index 1..16) and HUFFVAL */
static const uint8_t qe_std_bits[4][17] = {
	{ 0, 0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0 },             /* DC luminance   */
	{ 0, 0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d },          /* AC luminance   */
	{ 0, 0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0 },             /* DC chrominance */
	{ 0, 0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77 } };        /* AC chrominance */
static const uint8_t qe_std_ac_l[162] = {
	0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71,
	0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72,
	0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37,
	0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
	0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
	0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3,
	0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
	0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
	0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa };
static const uint8_t qe_std_ac_c[162] = {
	0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22,
	0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1,
	0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36,
	0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
	0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
	0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a,
	0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
	0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
	0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa };

/* ---------------------------------------------------------------- records */
struct QeGeo {                         /* one scan geometry of an image */
	const int16_t *coef[4];
	uint32_t wblk[4], hblk[4];
	uint8_t hs[4], vs[4];              /* blocks of the component in one MCU: 1 x 1 in a scan of one component */
	uint8_t sof_hv[4];                 /* the sampling factors the SOF gives */
	uint32_t mcux, mcuy, nblk, pad;
	uint8_t u_comp[QE_MAX_UNITS], u_h[QE_MAX_UNITS], u_v[QE_MAX_UNITS], pad1[2];
	uint64_t nunits;                   /* mcux * mcuy * nblk */
};

struct QeTab {                         /* one Huffman table: DC 0, AC 0, DC 1, AC 1 */
	uint64_t freq[257];                /* symbol counts (optimize)                        */
	uint32_t cs[256];                  /* (code << 8) | size, 0 = no code                 */
	uint8_t bits[17], val[256], pad[3];
	int32_t nval;
};

struct QeState {                       /* per image, written on the device */
	uint32_t geo, flags;               /* geometry in use; JPEGQS_ENCODE_RANGE           */
	uint64_t head_len;                 /* prefix + DQT + SOF + DHT + SOS                  */
	uint64_t total_bits, nraw;         /* entropy-coded bits; their bytes (last filled)  */
};

struct QeImg {                         /* per-image descriptor (host-made, copied by qe_setup) */
	QeGeo geo[2];                      /* 0: as sampled, 1: up-sampled chroma (coef_up, 1x1) */
	const jpegqs_cuda_status *run_status;
	int32_t upmode;                    /* 0 / 1: geometry 0 / 1; 2: run_status[i].upsampled decides;
	                                      3: geometry 0, NO_UP where run_status[i].upsampled is set */
	int32_t ncomp;
	uint32_t width, height;
	int32_t comp_id[4], qtbl[4], has_q[4];
	uint16_t quant[4][64];
	const uint8_t *prefix;
	uint64_t prefix_len;
	uint8_t *out;
	uint64_t cap;
	uint64_t *len;
	int32_t *status;
	int32_t index, optimize;
	/* workspace */
	QeState *st;
	QeTab *tab;                        /* [4]                                           */
	uint16_t *ulen;                    /* bits per unit                                 */
	uint64_t *tile;                    /* bits per tile, then their exclusive scan      */
	uint32_t *word;                    /* the unstuffed bits, first bit = bit 31        */
	uint32_t *ffc;                     /* 0xFF bytes per chunk, then their scan         */
};
static_assert(sizeof(QeImg) <= 2048 && sizeof(QeState) <= 1024 && 4096 + 4 * sizeof(QeTab) <= QE_FIXED, "fixed part");

/* ---------------------------------------------------------------- helpers shared by host and device */
HD static inline int qe_size(int v) {               /* bits of |v| (T.81 F.1.2.1 SSSS) */
	unsigned a = (unsigned)(v < 0 ? -v : v);
#ifdef __CUDA_ARCH__
	return 32 - __clz((int)a);
#else
	return a ? 32 - __builtin_clz(a) : 0;
#endif
}
HD static inline int qe_ctz64(uint64_t m) {
#ifdef __CUDA_ARCH__
	return __ffsll((long long)m) - 1;
#else
	return __builtin_ctzll(m);
#endif
}
HD static inline void qe_or(uint32_t *p, uint32_t v) {
#ifdef __CUDA_ARCH__
	atomicOr(p, v);
#else
	*p |= v;
#endif
}

/* the non-zero coefficients of a block as a mask in zig-zag order */
HD static inline uint64_t qe_zmask(const int16_t *blk) {
	uint64_t m = 0;
#ifdef __CUDA_ARCH__
	const int4 *p = reinterpret_cast<const int4 *>(blk);
#pragma unroll
	for (int j = 0; j < 8; j++) {
		int4 q = p[j];
		uint32_t w[4] = { (uint32_t)q.x, (uint32_t)q.y, (uint32_t)q.z, (uint32_t)q.w };
#pragma unroll
		for (int h = 0; h < 4; h++) {
			if (w[h] & 0xFFFFu) m |= 1ull << qe_zz_dev[8 * j + 2 * h];
			if (w[h] >> 16) m |= 1ull << qe_zz_dev[8 * j + 2 * h + 1];
		}
	}
#else
	for (int i = 0; i < 64; i++) if (blk[i]) m |= 1ull << qe_zz_host[i];
#endif
	return m;
}

/* block (bx, by) of unit k of MCU (mx, my), if it is a real block: its offset in the array */
HD static inline bool qe_real(const QeGeo &g, uint32_t k, uint64_t mx, uint64_t my, uint64_t *off) {
	int c = g.u_comp[k];
	uint64_t bx = mx * g.hs[c] + g.u_h[k], by = my * g.vs[c] + g.u_v[k];
	if (bx >= g.wblk[c] || by >= g.hblk[c]) return false;
	*off = (by * g.wblk[c] + bx) * 64;
	return true;
}

struct QeUnit { const int16_t *blk; int pred, tsel; };   /* blk NULL: padding block */

/* unit u of the scan: its block and its DC predictor, the DC of the last real block of its component
 * before it in MCU order (0 for the first) */
HD static inline QeUnit qe_locate(const QeGeo &g, uint64_t u) {
	QeUnit r;
	uint32_t k = (uint32_t)(u % g.nblk);
	uint64_t m = u / g.nblk, mx = m % g.mcux, my = m / g.mcux, off;
	int c = g.u_comp[k];
	r.tsel = c ? 1 : 0;
	r.blk = qe_real(g, k, mx, my, &off) ? g.coef[c] + off : NULL;
	r.pred = 0;
	for (int kk = (int)k - 1; kk >= 0; kk--)
		if (g.u_comp[kk] == c && qe_real(g, (uint32_t)kk, mx, my, &off)) { r.pred = g.coef[c][off]; return r; }
	if (m > 0) {
		m--; mx = m % g.mcux; my = m / g.mcux;
		for (int kk = (int)g.nblk - 1; kk >= 0; kk--)
			if (g.u_comp[kk] == c && qe_real(g, (uint32_t)kk, mx, my, &off)) { r.pred = g.coef[c][off]; return r; }
	}
	return r;
}

/* The symbols of one unit, in order, to sink.sym(table, symbol, value bits, value size): table =
 * 2 * tsel (+1 for AC).  Returns JPEGQS_ENCODE_RANGE for a DC difference of category > 11 or an AC
 * value of category > 10 (jq_write's "out of range"); such a value is coded at the largest category,
 * so the unit stays within 1665 bits. */
template <class S> HD static inline uint32_t qe_unit(const QeUnit &un, S &sink) {
	uint32_t bad = 0;
	int dc = un.blk ? un.blk[0] : un.pred, diff = dc - un.pred, s = qe_size(diff);
	if (s > 11) { bad = JPEGQS_ENCODE_RANGE; s = 11; }
	sink.sym(2 * un.tsel, s, (uint32_t)(diff + (diff >> 31)) & ((1u << s) - 1), s);
	int prev = 0;
	if (un.blk) {
		uint64_t m = qe_zmask(un.blk) & ~1ull;
		while (m) {
			int k = qe_ctz64(m);
			m &= m - 1;
			int run = k - prev - 1, v = un.blk[qe_nat(k)];
			prev = k;
			for (; run > 15; run -= 16) sink.sym(2 * un.tsel + 1, 0xF0, 0, 0);
			int z = qe_size(v);
			if (z > 10) { bad = JPEGQS_ENCODE_RANGE; z = 10; }
			sink.sym(2 * un.tsel + 1, run << 4 | z, (uint32_t)(v + (v >> 31)) & ((1u << z) - 1), z);
		}
	}
	if (prev != 63) sink.sym(2 * un.tsel + 1, 0x00, 0, 0);
	return bad;
}

struct QeLenSink {
	const uint32_t *cs[4]; uint32_t n;
	HD void sym(int t, int s, uint32_t, int nv) { n += (cs[t][s] & 255) + (uint32_t)nv; }
};

/* bits into the word buffer from bit offset o on: full words by plain stores (the unit owns them),
 * the first word (when o is not word-aligned) and the last partial one by OR (shared) */
struct QeEmitSink {
	const uint32_t *cs[4];
	uint32_t *w; uint64_t base; uint64_t acc; int nacc; bool shared;
	HD void put(uint32_t v, int n) {
		acc = (acc << n) | v; nacc += n;
		if (nacc >= 32) {
			uint32_t x = (uint32_t)(acc >> (nacc - 32));
			if (shared) qe_or(w + (base >> 5), x); else w[base >> 5] = x;
			shared = false; nacc -= 32; base += 32;
		}
	}
	HD void sym(int t, int s, uint32_t vb, int nv) {
		uint32_t c = cs[t][s];
		put((c >> 8) << nv | vb, (int)(c & 255) + nv);
	}
	HD void finish() {
		if (nacc) qe_or(w + (base >> 5), (uint32_t)((acc & ((1ull << nacc) - 1)) << (32 - nacc)));
	}
};

HD static inline void qe_emit_unit(const QeGeo &g, uint64_t u, uint64_t o, const uint32_t *const *cs, uint32_t *word,
		uint64_t total) {
	QeEmitSink e;
	for (int t = 0; t < 4; t++) e.cs[t] = cs[t];
	e.w = word; e.base = o & ~31ull; e.acc = 0; e.nacc = (int)(o & 31); e.shared = (o & 31) != 0;
	qe_unit(qe_locate(g, u), e);
	if (u + 1 == g.nunits) {                         /* the last byte is filled with 1-bits */
		int pad = (int)((8 - (total & 7)) & 7);
		if (pad) e.put((1u << pad) - 1, pad);
	}
	e.finish();
}

/* ---------------------------------------------------------------- tables: jq_write's ehuff_codes / ehuff_optimal */
HD static inline void qe_codes(QeTab *t) {          /* T.81 C.2 */
	uint32_t code = 0; int k = 0;
	for (int i = 0; i < 256; i++) t->cs[i] = 0;
	for (int l = 1; l <= 16; l++) {
		for (int i = 0; i < t->bits[l] && k < 256; i++, k++) t->cs[t->val[k]] = code++ << 8 | (uint32_t)l;
		code <<= 1;
	}
}

/* the candidate ehuff_optimal's "freq[i] && freq[i] <= v" scan picks: the smallest frequency, the last
 * index among equals, none above the sentinel.  nl lanes of a warp scan strided and reduce. */
HD static inline int qe_pick(const uint64_t *f, int excl, int lane, int nl) {
	uint64_t bv = QE_SENT + 1; int bi = -1;
	for (int i = lane; i <= 256; i += nl) {
		uint64_t x = f[i];
		if (x && x <= QE_SENT && i != excl && (x < bv || (x == bv && i > bi))) { bv = x; bi = i; }
	}
#ifdef __CUDA_ARCH__
	if (nl > 1)
		for (int o = 16; o; o >>= 1) {
			uint64_t ov = __shfl_xor_sync(0xFFFFFFFFu, bv, o);
			int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
			if (ov < bv || (ov == bv && oi > bi)) { bv = ov; bi = oi; }
		}
#endif
	return bi;
}

/* optimal code lengths limited to 16 bits (T.81 K.2, figures K.1 - K.4), exactly as jq_write's
 * ehuff_optimal: the reserved symbol 256, ties broken by the last index, the 10^9 sentinel, the
 * K.3 length limiting and HUFFVAL in (code length, symbol) order.  Scratch arrays of 257 entries. */
HD static inline void qe_optimal(QeTab *t, uint64_t *freq, int *codesize, int *others, int lane, int nl) {
	for (int i = lane; i < 257; i += nl) { freq[i] = t->freq[i]; codesize[i] = 0; others[i] = -1; }
#ifdef __CUDA_ARCH__
	__syncwarp();
#endif
	if (lane == 0) freq[256] = 1;
#ifdef __CUDA_ARCH__
	__syncwarp();
#endif
	for (;;) {
		int c1 = qe_pick(freq, -1, lane, nl), c2 = qe_pick(freq, c1, lane, nl);
		if (c2 < 0) break;
		if (lane == 0) {
			freq[c1] += freq[c2]; freq[c2] = 0;
			for (codesize[c1]++; others[c1] >= 0; codesize[c1]++) c1 = others[c1];
			others[c1] = c2;
			for (codesize[c2]++; others[c2] >= 0; codesize[c2]++) c2 = others[c2];
		}
#ifdef __CUDA_ARCH__
		__syncwarp();
#endif
	}
	if (lane == 0) {
		int bits[33], i, j, k;
		for (i = 0; i < 33; i++) bits[i] = 0;
		for (i = 0; i <= 256; i++) if (codesize[i]) bits[codesize[i] > 32 ? 32 : codesize[i]]++;
		for (i = 32; i > 16; i--) while (bits[i] > 0) {
			for (j = i - 2; j > 0 && bits[j] == 0; j--);
			bits[i] -= 2; bits[i - 1]++; bits[j + 1] += 2; bits[j]--;
		}
		while (i > 0 && bits[i] == 0) i--;
		bits[i]--;                                   /* drop the reserved code point */
		t->bits[0] = 0;
		for (i = 1; i <= 16; i++) t->bits[i] = (uint8_t)bits[i];
		for (k = 0, i = 1; i <= 32; i++) for (j = 0; j < 256; j++) if (codesize[j] == i) t->val[k++] = (uint8_t)j;
		t->nval = k;
	}
#ifdef __CUDA_ARCH__
	__syncwarp();
#endif
}

/* the four tables' source for optimize == 0 */
struct QeStd { uint8_t bits[4][17]; uint8_t val[4][162]; int32_t nval[4]; };

HD static inline void qe_set_std(QeTab *t, const QeStd &s, int w) {
	for (int i = 0; i < 17; i++) t->bits[i] = s.bits[w][i];
	for (int i = 0; i < s.nval[w]; i++) t->val[i] = s.val[w][i];
	t->nval = s.nval[w];
}

/* ---------------------------------------------------------------- the header segments */
struct QeOut {
	uint8_t *p; uint64_t cap, n;
	HD void b(unsigned v) { if (n < cap) p[n] = (uint8_t)v; n++; }
	HD void w(unsigned v) { b(v >> 8); b(v & 255); }
};

/* DQT for every table in use, then SOF0 / SOF1 (SOF2 when progressive) */
HD static inline void qe_frame(const QeImg &im, const QeGeo &g, QeOut &o, bool progressive) {
	int nc = im.ncomp, sof = 0xC0;
	unsigned written = 0;
	for (int k = 0; k < nc; k++) {
		int tq = im.qtbl[k] & 3, prec = 0;
		if (!im.has_q[k] || (written >> tq & 1)) continue;
		written |= 1u << tq;
		for (int i = 0; i < 64; i++) if (im.quant[k][i] > 255) prec = 1;
		if (prec) sof = 0xC1;
		o.w(0xFFDB); o.w(2 + 1 + (prec ? 128 : 64)); o.b((unsigned)(prec << 4 | tq));
		for (int i = 0; i < 64; i++) { unsigned v = im.quant[k][qe_nat(i)]; if (prec) o.w(v); else o.b(v); }
	}
	o.w(0xFF00 | (progressive ? 0xC2 : sof)); o.w(8 + 3 * nc); o.b(8);
	o.w(im.height); o.w(im.width); o.b((unsigned)nc);
	for (int k = 0; k < nc; k++) { o.b((unsigned)im.comp_id[k]); o.b((unsigned)g.sof_hv[k]); o.b((unsigned)im.qtbl[k]); }
}

/* DQT for every table in use, SOF0 / SOF1, DHT, SOS - jq_write's order - written from prefix_len on
 * (nothing at or past cap).  Returns the header length, prefix included. */
HD static inline uint64_t qe_header(const QeImg &im, const QeGeo &g, const QeTab *tab, uint8_t *out, uint64_t cap) {
	QeOut o = { out, cap, im.prefix_len };
	int nc = im.ncomp, nt = nc > 1 ? 2 : 1;
	qe_frame(im, g, o, false);
	for (int i = 0; i < nt; i++) for (int a = 0; a < 2; a++) {
		const QeTab &t = tab[2 * i + a];
		o.w(0xFFC4); o.w(2 + 1 + 16 + t.nval); o.b((unsigned)(a << 4 | i));
		for (int l = 1; l <= 16; l++) o.b(t.bits[l]);
		for (int l = 0; l < t.nval; l++) o.b(t.val[l]);
	}
	o.w(0xFFDA); o.w(6 + 2 * nc); o.b((unsigned)nc);
	for (int k = 0; k < nc; k++) { o.b((unsigned)im.comp_id[k]); o.b(k ? 0x11u : 0x00u); }
	o.b(0); o.b(63); o.b(0);
	return o.n;
}

/* ---------------------------------------------------------------- byte passes: rules shared by host and device */
HD static inline unsigned qe_byte(const uint32_t *w, uint64_t j) { return (w[j >> 2] >> (24 - 8 * (j & 3))) & 255; }

/* the 0xFF bytes among unstuffed bytes [j0, j1) */
HD static inline uint32_t qe_ffs(const uint32_t *w, uint64_t j0, uint64_t j1) {
	uint32_t n = 0;
	for (uint64_t j = j0; j < j1; j++) n += qe_byte(w, j) == 0xFF;
	return n;
}
/* bytes [j0, j1) stuffed to out from position pos on (nothing at or past cap) */
HD static inline void qe_stuff(const uint32_t *w, uint64_t j0, uint64_t j1, uint8_t *out, uint64_t cap, uint64_t pos) {
	for (uint64_t j = j0; j < j1; j++) {
		unsigned c = qe_byte(w, j);
		if (pos < cap) out[pos] = (uint8_t)c;
		pos++;
		if (c == 0xFF) { if (pos < cap) out[pos] = 0; pos++; }
	}
}

/* ---------------------------------------------------------------- kernels */
struct QeSetupPack {
	QeImg img[QE_PACK];
	int n;
};
static_assert(sizeof(QeSetupPack) <= 32000, "QeSetupPack exceeds the kernel parameter space");

struct QePtrs { const QeImg *img[QE_PACK]; int n; };

HD static inline const QeGeo &qe_geo(const QeImg &im) { return im.geo[im.st->geo]; }

/* blockIdx.x = image: descriptor, geometry choice, state, histograms */
__global__ void __launch_bounds__(256) qe_setup_kernel(const __grid_constant__ QeSetupPack p) {
	int i = blockIdx.x;
	if (i >= p.n) return;
	const QeImg &im = p.img[i];
	if (threadIdx.x == 0) {
		*reinterpret_cast<QeImg *>(reinterpret_cast<char *>(im.st) - 2048) = im;
		QeState s = {};
		bool dev_up = im.upmode >= 2 && im.run_status[im.index].upsampled != 0;
		s.geo = im.upmode == 2 ? (dev_up ? 1u : 0u) : im.upmode == 3 ? 0u : (uint32_t)im.upmode;
		if (im.upmode == 3 && dev_up) s.flags = JPEGQS_ENCODE_NO_UP;     /* up-sampled, but no coef_up given */
		*im.st = s;
	}
	for (int j = threadIdx.x; j < 4 * 257; j += blockDim.x) im.tab[j / 257].freq[j % 257] = 0;
}

struct QeCountSink {
	uint32_t (*h)[257];
	__device__ void sym(int t, int s, uint32_t, int) { atomicAdd(&h[t][s], 1u); }
};

/* optimize: per tile, the symbols of its units into shared histograms, then into the image's */
__global__ void __launch_bounds__(QE_T) qe_count_kernel(const __grid_constant__ QePtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QeImg &im = *P.img[blockIdx.y];
	const QeGeo &g = qe_geo(im);
	uint64_t u0 = (uint64_t)blockIdx.x * QE_T;
	if (u0 >= g.nunits) return;
	__shared__ uint32_t h[4][257];
	for (int j = threadIdx.x; j < 4 * 257; j += QE_T) h[j / 257][j % 257] = 0;
	__syncthreads();
	uint64_t u = u0 + threadIdx.x;
	uint32_t bad = 0;
	if (u < g.nunits) { QeCountSink s = { h }; bad = qe_unit(qe_locate(g, u), s); }
	if (bad) atomicOr(&im.st->flags, bad);
	__syncthreads();
	for (int j = threadIdx.x; j < 4 * 257; j += QE_T) {
		uint32_t v = h[j / 257][j % 257];
		if (v) atomicAdd(reinterpret_cast<unsigned long long *>(&im.tab[j / 257].freq[j % 257]), (unsigned long long)v);
	}
}

/* blockIdx.x = image, warp w = table w: the standard or the optimal table and its codes; then the
 * prefix copy and the header segments */
__global__ void __launch_bounds__(128) qe_table_kernel(const __grid_constant__ QePtrs P, const __grid_constant__ QeStd std) {
	if ((int)blockIdx.x >= P.n) return;
	const QeImg &im = *P.img[blockIdx.x];
	__shared__ uint64_t s_freq[4][257];
	__shared__ int s_size[4][257], s_oth[4][257];
	int w = threadIdx.x >> 5, lane = threadIdx.x & 31, nt = im.ncomp > 1 ? 2 : 1;
	QeTab *t = im.tab + w;
	if (w / 2 < nt) {
		if (im.optimize) qe_optimal(t, s_freq[w], s_size[w], s_oth[w], lane, 32);
		else if (lane == 0) qe_set_std(t, std, w);
		__syncwarp();
		if (lane == 0) qe_codes(t);
	}
	for (uint64_t j = threadIdx.x; j < im.prefix_len && j < im.cap; j += blockDim.x) im.out[j] = im.prefix[j];
	__syncthreads();
	if (threadIdx.x == 0) im.st->head_len = qe_header(im, qe_geo(im), im.tab, im.out, im.cap);
}

/* per tile: every unit's bit length, the tile's sum */
__global__ void __launch_bounds__(QE_T) qe_len_kernel(const __grid_constant__ QePtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QeImg &im = *P.img[blockIdx.y];
	const QeGeo &g = qe_geo(im);
	uint64_t u0 = (uint64_t)blockIdx.x * QE_T;
	if (u0 >= g.nunits) return;
	__shared__ uint32_t s_cs[4][256];
	for (int j = threadIdx.x; j < 4 * 256; j += QE_T) s_cs[j >> 8][j & 255] = im.tab[j >> 8].cs[j & 255];
	__syncthreads();
	uint64_t u = u0 + threadIdx.x;
	uint32_t n = 0, bad = 0;
	if (u < g.nunits) {
		QeLenSink s = { { s_cs[0], s_cs[1], s_cs[2], s_cs[3] }, 0 };
		bad = qe_unit(qe_locate(g, u), s);
		n = s.n;
		im.ulen[u] = (uint16_t)n;
	}
	if (bad) atomicOr(&im.st->flags, bad);
	typedef cub::BlockReduce<uint32_t, QE_T> R;
	__shared__ typename R::TempStorage tmp;
	uint32_t sum = R(tmp).Sum(n);
	if (threadIdx.x == 0) im.tile[blockIdx.x] = sum;
}

/* per image: exclusive scan of the tile sums; total bits */
__global__ void __launch_bounds__(QE_SCAN_T) qe_tscan_kernel(const __grid_constant__ QePtrs P) {
	if ((int)blockIdx.x >= P.n) return;
	const QeImg &im = *P.img[blockIdx.x];
	const QeGeo &g = qe_geo(im);
	uint64_t ntile = (g.nunits + QE_T - 1) / QE_T, carry = 0;
	typedef cub::BlockScan<uint64_t, QE_SCAN_T> S;
	__shared__ typename S::TempStorage tmp;
	for (uint64_t base = 0; base < ntile; base += QE_SCAN_T) {
		uint64_t t = base + threadIdx.x, v = t < ntile ? im.tile[t] : 0, ex, agg;
		S(tmp).ExclusiveSum(v, ex, agg);
		if (t < ntile) im.tile[t] = carry + ex;
		carry += agg;
		__syncthreads();
	}
	if (threadIdx.x == 0) { im.st->total_bits = carry; im.st->nraw = (carry + 7) >> 3; }
}

/* the words the bits will occupy, and one more, set to zero */
__global__ void __launch_bounds__(256) qe_zero_kernel(const __grid_constant__ QePtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QeImg &im = *P.img[blockIdx.y];
	uint64_t nw = (im.st->total_bits + 31) / 32 + 1;
	for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nw; j += (uint64_t)gridDim.x * blockDim.x) im.word[j] = 0;
}

/* per tile: the units' bit offsets (tile offset + scan inside the tile), their bits */
__global__ void __launch_bounds__(QE_T) qe_emit_kernel(const __grid_constant__ QePtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QeImg &im = *P.img[blockIdx.y];
	const QeGeo &g = qe_geo(im);
	uint64_t u0 = (uint64_t)blockIdx.x * QE_T;
	if (u0 >= g.nunits) return;
	__shared__ uint32_t s_cs[4][256];
	for (int j = threadIdx.x; j < 4 * 256; j += QE_T) s_cs[j >> 8][j & 255] = im.tab[j >> 8].cs[j & 255];
	uint64_t u = u0 + threadIdx.x;
	uint32_t n = u < g.nunits ? im.ulen[u] : 0, ex;
	typedef cub::BlockScan<uint32_t, QE_T> S;
	__shared__ typename S::TempStorage tmp;
	S(tmp).ExclusiveSum(n, ex);
	__syncthreads();
	if (u < g.nunits) {
		const uint32_t *cs[4] = { s_cs[0], s_cs[1], s_cs[2], s_cs[3] };
		qe_emit_unit(g, u, im.tile[blockIdx.x] + ex, cs, im.word, im.st->total_bits);
	}
}

/* per chunk of QE_CHUNK unstuffed bytes: its 0xFF bytes */
__global__ void __launch_bounds__(QE_BT) qe_ffcount_kernel(const __grid_constant__ QePtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QeImg &im = *P.img[blockIdx.y];
	uint64_t nraw = im.st->nraw, c0 = (uint64_t)blockIdx.x * QE_CHUNK;
	if (c0 >= nraw) return;
	uint64_t j0 = c0 + threadIdx.x * 16, j1 = j0 + 16 < nraw ? j0 + 16 : nraw;
	uint32_t n = j0 < nraw ? qe_ffs(im.word, j0, j1) : 0;
	typedef cub::BlockReduce<uint32_t, QE_BT> R;
	__shared__ typename R::TempStorage tmp;
	uint32_t sum = R(tmp).Sum(n);
	if (threadIdx.x == 0) im.ffc[blockIdx.x] = sum;
}

/* per image: exclusive scan of the chunk counts; file length, status, EOI */
__global__ void __launch_bounds__(QE_SCAN_T) qe_fscan_kernel(const __grid_constant__ QePtrs P) {
	if ((int)blockIdx.x >= P.n) return;
	const QeImg &im = *P.img[blockIdx.x];
	const QeState *st = im.st;
	uint64_t nchunk = (st->nraw + QE_CHUNK - 1) / QE_CHUNK, carry = 0;
	typedef cub::BlockScan<uint64_t, QE_SCAN_T> S;
	__shared__ typename S::TempStorage tmp;
	for (uint64_t base = 0; base < nchunk; base += QE_SCAN_T) {
		uint64_t c = base + threadIdx.x, v = c < nchunk ? im.ffc[c] : 0, ex, agg;
		S(tmp).ExclusiveSum(v, ex, agg);
		if (c < nchunk) im.ffc[c] = (uint32_t)(carry + ex);
		carry += agg;
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		uint64_t end = st->head_len + st->nraw + carry, L = end + 2;
		int32_t flags = (int32_t)st->flags;
		if (L > im.cap) flags |= JPEGQS_ENCODE_OVERFLOW;
		else { im.out[end] = 0xFF; im.out[end + 1] = 0xD9; }
		*im.len = L;
		*im.status = flags;
	}
}

/* per chunk: its bytes stuffed to the output */
__global__ void __launch_bounds__(QE_BT) qe_copy_kernel(const __grid_constant__ QePtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QeImg &im = *P.img[blockIdx.y];
	uint64_t nraw = im.st->nraw, c0 = (uint64_t)blockIdx.x * QE_CHUNK;
	if (c0 >= nraw) return;
	uint64_t j0 = c0 + threadIdx.x * 16, j1 = j0 + 16 < nraw ? j0 + 16 : nraw;
	uint32_t n = j0 < nraw ? qe_ffs(im.word, j0, j1) : 0, ex;
	typedef cub::BlockScan<uint32_t, QE_BT> S;
	__shared__ typename S::TempStorage tmp;
	S(tmp).ExclusiveSum(n, ex);
	if (j0 < nraw) qe_stuff(im.word, j0, j1, im.out, im.cap, im.st->head_len + j0 + im.ffc[blockIdx.x] + ex);
}

/* ---------------------------------------------------------------- host: checks, sizes, launches */
struct jpegqs_cuda_ctx;
void qs_ctx_decode_info(jpegqs_cuda_ctx *ctx, int *device, cudaStream_t *stream, int *sub_bytes);
void qs_ctx_decode_done(jpegqs_cuda_ctx *ctx, int launches, const char *err);
extern "C" void qs_set_host_error(const char *msg);

static size_t qe_a256(size_t x) { return (x + 255) & ~(size_t)255; }

/* geometry 1 exists for images UPSAMPLE_UV can turn into three 1x1 components (YCbCr, chroma 1x1, luma not) */
static bool qe_can_up(const jpegqs_cuda_image *im) {
	const jpegqs_cuda_comp *c = im->comp;
	return im->ncomp == 3 && im->is_ycbcr && c[1].h_samp == 1 && c[1].v_samp == 1 && c[2].h_samp == 1 && c[2].v_samp == 1 &&
		(c[0].h_samp != 1 || c[0].v_samp != 1);
}

/* the geometries of an image: 0 as sampled, 1 up-sampled; returns 0 or a message */
static const char *qe_geometry(const jpegqs_cuda_image *im, QeGeo *g0, QeGeo *g1, bool *up_ok) {
	int nc = im->ncomp, maxh = 1, maxv = 1;
	memset(g0, 0, sizeof(*g0)); memset(g1, 0, sizeof(*g1));
	if (nc < 1 || nc > 4) return "ncomp outside 1..4";
	if (!im->image_width || !im->image_height || im->image_width > 65535 || im->image_height > 65535) return "image size outside 1..65535";
	for (int c = 0; c < nc; c++) {
		const jpegqs_cuda_comp &cc = im->comp[c];
		if (cc.h_samp < 1 || cc.h_samp > 4 || cc.v_samp < 1 || cc.v_samp > 4) return "sampling factor outside 1..4";
		if (cc.rows || cc.rows_up) return "rows / rows_up set";
		maxh = cc.h_samp > maxh ? cc.h_samp : maxh; maxv = cc.v_samp > maxv ? cc.v_samp : maxv;
	}
	uint32_t nb = 0;
	for (int c = 0; c < nc; c++) {
		const jpegqs_cuda_comp &cc = im->comp[c];
		uint64_t wb = ((uint64_t)im->image_width * cc.h_samp + 8 * maxh - 1) / (8 * maxh);
		uint64_t hb = ((uint64_t)im->image_height * cc.v_samp + 8 * maxv - 1) / (8 * maxv);
		if (cc.wblk != wb || cc.hblk != hb) return "wblk / hblk are not libjpeg's for this image size";
		g0->coef[c] = cc.coef; g0->wblk[c] = cc.wblk; g0->hblk[c] = cc.hblk;
		/* a scan of one component is not interleaved: its MCU is one block, whatever the factors (A.2.2) */
		g0->hs[c] = nc == 1 ? 1 : (uint8_t)cc.h_samp; g0->vs[c] = nc == 1 ? 1 : (uint8_t)cc.v_samp;
		g0->sof_hv[c] = (uint8_t)(cc.h_samp << 4 | cc.v_samp);
		for (int v = 0; v < g0->vs[c]; v++) for (int h = 0; h < g0->hs[c]; h++) {
			if (nb >= QE_MAX_UNITS) return "more than 10 blocks per MCU";
			g0->u_comp[nb] = (uint8_t)c; g0->u_h[nb] = (uint8_t)h; g0->u_v[nb] = (uint8_t)v; nb++;
		}
	}
	g0->nblk = nb;
	g0->mcux = nc == 1 ? im->comp[0].wblk : (uint32_t)(((uint64_t)im->image_width + 8 * maxh - 1) / (8 * maxh));
	g0->mcuy = nc == 1 ? im->comp[0].hblk : (uint32_t)(((uint64_t)im->image_height + 8 * maxv - 1) / (8 * maxv));
	g0->nunits = (uint64_t)g0->mcux * g0->mcuy * nb;
	*up_ok = qe_can_up(im);
	if (*up_ok) {
		for (int c = 0; c < 3; c++) {
			g1->coef[c] = c ? im->comp[c].coef_up : im->comp[0].coef;
			g1->wblk[c] = im->comp[0].wblk; g1->hblk[c] = im->comp[0].hblk; g1->hs[c] = g1->vs[c] = 1; g1->sof_hv[c] = 0x11;
			g1->u_comp[c] = (uint8_t)c;
		}
		g1->nblk = 3;
		g1->mcux = (im->image_width + 7) / 8; g1->mcuy = (im->image_height + 7) / 8;
		g1->nunits = (uint64_t)g1->mcux * g1->mcuy * 3;
	}
	return NULL;
}

/* the units a workspace / bound must cover: the larger geometry */
static uint64_t qe_max_units(const QeGeo &g0, const QeGeo &g1, bool up_ok) {
	return up_ok && g1.nunits > g0.nunits ? g1.nunits : g0.nunits;
}

struct QeSizes { uint64_t units, tiles, words, chunks; size_t bytes; };
static QeSizes qe_sizes(uint64_t U) {
	QeSizes s;
	s.units = U;
	s.tiles = (U + QE_T - 1) / QE_T;
	s.words = (U * QE_BLOCK_BITS + 31) / 32 + 2;
	s.chunks = (4 * s.words + QE_CHUNK - 1) / QE_CHUNK;
	s.bytes = QE_FIXED + qe_a256(2 * U) + qe_a256(8 * s.tiles) + qe_a256(4 * s.words) + qe_a256(4 * s.chunks);
	return s;
}

extern "C" int jpegqs_cuda_encode_bound(const jpegqs_cuda_image *img, size_t prefix_len, size_t *bytes) {
	if (!img || !bytes) { qs_set_host_error("jpegqs_cuda_encode_bound: NULL argument"); return JPEGQS_ERR_ARG; }
	QeGeo g0, g1; bool up;
	const char *e = qe_geometry(img, &g0, &g1, &up);
	if (e) { char m[256]; snprintf(m, sizeof(m), "jpegqs_cuda_encode_bound: %s", e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
	uint64_t U = qe_max_units(g0, g1, up);
	*bytes = prefix_len + QE_HEAD_MAX + 2 * ((U * QE_BLOCK_BITS + 7) / 8);
	return 0;
}

extern "C" int jpegqs_cuda_encode_workspace_bytes(int n, const jpegqs_cuda_image *imgs, int optimize, size_t *bytes) {
	(void)optimize;
	if (n < 0 || !bytes || (n && !imgs)) { qs_set_host_error("jpegqs_cuda_encode_workspace_bytes: NULL argument"); return JPEGQS_ERR_ARG; }
	size_t total = 0;
	for (int i = 0; i < n; i++) {
		QeGeo g0, g1; bool up;
		const char *e = qe_geometry(&imgs[i], &g0, &g1, &up);
		if (e) { char m[256]; snprintf(m, sizeof(m), "jpegqs_cuda_encode_workspace_bytes: image %d: %s", i, e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
		total += qe_sizes(qe_max_units(g0, g1, up)).bytes;
	}
	*bytes = total;
	return 0;
}

/* checks image i with its head and output and fills its descriptor (pointers; workspace not yet) */
static const char *qe_check(const jpegqs_cuda_image *im, const jpegqs_cuda_jpeg_head *hd, bool status_path, int optimize,
		QeImg *d, QeSizes *sz) {
	memset(d, 0, sizeof(*d));
	bool up;
	const char *e = qe_geometry(im, &d->geo[0], &d->geo[1], &up);
	if (e) return e;
	int nc = im->ncomp;
	for (int c = 0; c < nc; c++) {
		if (!im->comp[c].coef) return "coef NULL";
		if ((uintptr_t)im->comp[c].coef & 15) return "coef not 16-byte aligned";
	}
	bool have_up = up && im->comp[1].coef_up && im->comp[2].coef_up;
	if (have_up) for (int c = 1; c < 3; c++) if ((uintptr_t)im->comp[c].coef_up & 15) return "coef_up not 16-byte aligned";
	if (status_path) d->upmode = have_up ? 2 : up ? 3 : 0;
	else if (im->upsampled) {
		if (!up) return "upsampled set on an image UPSAMPLE_UV cannot up-sample";
		if (!have_up) return "upsampled set but coef_up NULL";
		d->upmode = 1;
	} else d->upmode = 0;
	if (!hd) return "heads NULL";
	if (hd->prefix_len && !hd->prefix_dev) return "prefix_dev NULL";
	for (int c = 0; c < nc; c++) {
		if (hd->comp_id[c] < 0 || hd->comp_id[c] > 255) return "comp_id outside 0..255";
		if (hd->quant_tbl[c] < 0 || hd->quant_tbl[c] > 3) return "quant_tbl outside 0..3";
		d->comp_id[c] = hd->comp_id[c]; d->qtbl[c] = hd->quant_tbl[c]; d->has_q[c] = im->comp[c].has_qtbl != 0;
		memcpy(d->quant[c], im->comp[c].quant, sizeof(d->quant[c]));
	}
	d->ncomp = nc; d->width = im->image_width; d->height = im->image_height;
	d->prefix = hd->prefix_dev; d->prefix_len = hd->prefix_len;
	d->optimize = optimize != 0;
	*sz = qe_sizes(qe_max_units(d->geo[0], d->geo[1], up));
	return NULL;
}

static void qe_carve(QeImg *d, const QeSizes &sz, char *w) {
	d->st = reinterpret_cast<QeState *>(w + 2048);
	d->tab = reinterpret_cast<QeTab *>(w + 4096);
	w += QE_FIXED;
	d->ulen = reinterpret_cast<uint16_t *>(w); w += qe_a256(2 * sz.units);
	d->tile = reinterpret_cast<uint64_t *>(w); w += qe_a256(8 * sz.tiles);
	d->word = reinterpret_cast<uint32_t *>(w); w += qe_a256(4 * sz.words);
	d->ffc = reinterpret_cast<uint32_t *>(w);
}

static QeStd qe_std() {
	QeStd s;
	memset(&s, 0, sizeof(s));
	memcpy(s.bits, qe_std_bits, sizeof(s.bits));
	for (int i = 0; i < 12; i++) s.val[0][i] = s.val[2][i] = (uint8_t)i;
	memcpy(s.val[1], qe_std_ac_l, 162); memcpy(s.val[3], qe_std_ac_c, 162);
	s.nval[0] = s.nval[2] = 12; s.nval[1] = s.nval[3] = 162;
	return s;
}

#define QE_CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	snprintf(msg, sizeof(msg), "%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
	qs_ctx_decode_done(ctx, launches, msg); return JPEGQS_ERR_CUDA; } } while (0)

extern "C" int jpegqs_cuda_encode_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_image *imgs,
		const jpegqs_cuda_jpeg_head *heads, int optimize, const jpegqs_cuda_status *run_status_dev,
		uint8_t *const *out_dev, const size_t *out_cap, uint64_t *len_dev, int32_t *status_dev,
		void *workspace, size_t workspace_bytes, void *stream) {
	char msg[512] = "";
	int launches = 0;
	if (!ctx) return JPEGQS_ERR_ARG;
	int device, unused; cudaStream_t st;
	qs_ctx_decode_info(ctx, &device, &st, &unused);
	if (stream) st = (cudaStream_t)stream;
	if (n < 0 || (n && (!imgs || !heads || !out_dev || !out_cap || !len_dev || !status_dev || !workspace))) {
		qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_encode_async: NULL argument"); return JPEGQS_ERR_ARG;
	}
	if ((uintptr_t)workspace & 255) { qs_ctx_decode_done(ctx, 0, "jpegqs_cuda_encode_async: workspace not 256-byte aligned"); return JPEGQS_ERR_ARG; }
	std::vector<QeImg> desc((size_t)n);
	std::vector<QeSizes> sizes((size_t)n);
	size_t need = 0;
	for (int i = 0; i < n; i++) {
		const char *e = qe_check(&imgs[i], &heads[i], run_status_dev != NULL, optimize, &desc[i], &sizes[i]);
		if (!e && !out_dev[i]) e = "out_dev entry NULL";
		if (!e && out_cap[i] < heads[i].prefix_len) e = "out_cap smaller than prefix_len";
		if (e) { snprintf(msg, sizeof(msg), "jpegqs_cuda_encode_async: image %d: %s", i, e); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
		need += sizes[i].bytes;
	}
	if (workspace_bytes < need) {
		snprintf(msg, sizeof(msg), "jpegqs_cuda_encode_async: workspace of %zu bytes, %zu needed", workspace_bytes, need);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	if (!n) { qs_ctx_decode_done(ctx, 0, ""); return 0; }
	QE_CK(cudaSetDevice(device));
	char *w = (char *)workspace;
	for (int i = 0; i < n; i++) {
		QeImg &d = desc[i];
		qe_carve(&d, sizes[i], w); w += sizes[i].bytes;
		d.run_status = run_status_dev; d.index = i;
		d.out = out_dev[i]; d.cap = out_cap[i]; d.len = len_dev + i; d.status = status_dev + i;
	}
	QeStd stdt = qe_std();
	for (int g0 = 0; g0 < n; g0 += QE_PACK) {
		int g = n - g0 < QE_PACK ? n - g0 : QE_PACK;
		std::unique_ptr<QeSetupPack> hold(new QeSetupPack());   /* per call (~30 KB: not on the stack) */
		QeSetupPack &pack = *hold;
		QePtrs P;
		memset(&pack, 0, sizeof(pack)); memset(&P, 0, sizeof(P));
		pack.n = g; P.n = g;
		uint64_t maxtile = 1, maxchunk = 1;
		for (int j = 0; j < g; j++) {
			pack.img[j] = desc[g0 + j];
			P.img[j] = reinterpret_cast<const QeImg *>(reinterpret_cast<const char *>(desc[g0 + j].st) - 2048);
			if (sizes[g0 + j].tiles > maxtile) maxtile = sizes[g0 + j].tiles;
			if (sizes[g0 + j].chunks > maxchunk) maxchunk = sizes[g0 + j].chunks;
		}
		if (maxtile > 0x7FFFFFFFull || maxchunk > 0x7FFFFFFFull) { qs_ctx_decode_done(ctx, launches, "jpegqs_cuda_encode_async: image too large"); return JPEGQS_ERR_ARG; }
		unsigned zero_blocks = (unsigned)(maxchunk < 4096 ? maxchunk : 4096);
		qe_setup_kernel<<<g, 256, 0, st>>>(pack); launches++;
		if (optimize) { qe_count_kernel<<<dim3((unsigned)maxtile, g), QE_T, 0, st>>>(P); launches++; }
		qe_table_kernel<<<g, 128, 0, st>>>(P, stdt); launches++;
		qe_len_kernel<<<dim3((unsigned)maxtile, g), QE_T, 0, st>>>(P); launches++;
		qe_tscan_kernel<<<g, QE_SCAN_T, 0, st>>>(P); launches++;
		qe_zero_kernel<<<dim3(zero_blocks, g), 256, 0, st>>>(P); launches++;
		qe_emit_kernel<<<dim3((unsigned)maxtile, g), QE_T, 0, st>>>(P); launches++;
		qe_ffcount_kernel<<<dim3((unsigned)maxchunk, g), QE_BT, 0, st>>>(P); launches++;
		qe_fscan_kernel<<<g, QE_SCAN_T, 0, st>>>(P); launches++;
		qe_copy_kernel<<<dim3((unsigned)maxchunk, g), QE_BT, 0, st>>>(P); launches++;
		QE_CK(cudaGetLastError());
	}
	qs_ctx_decode_done(ctx, launches, "");
	return 0;
}

/* ---------------------------------------------------------------- the CPU model */
extern "C" int jpegqs_cuda_encode_model(const jpegqs_cuda_image *img, const jpegqs_cuda_jpeg_head *head, int optimize,
		uint8_t *out, size_t cap, uint64_t *len, int32_t *status) {
	if (!img || !head || !out || !len || !status) { qs_set_host_error("jpegqs_cuda_encode_model: NULL argument"); return JPEGQS_ERR_ARG; }
	QeImg im; QeSizes sz;
	const char *e = qe_check(img, head, false, optimize, &im, &sz);
	if (!e && cap < head->prefix_len) e = "cap smaller than prefix_len";
	if (e) { char m[256]; snprintf(m, sizeof(m), "jpegqs_cuda_encode_model: %s", e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
	QeState st = {};
	st.geo = (uint32_t)im.upmode;                    /* the model has no run status: 0 or 1 */
	im.st = &st;
	const QeGeo &g = im.geo[st.geo];
	std::vector<QeTab> tab(4);
	memset(tab.data(), 0, 4 * sizeof(QeTab));
	im.tab = tab.data();
	/* qe_count */
	if (optimize) {
		struct { QeTab *t; void sym(int k, int s, uint32_t, int) { t[k].freq[s]++; } } cnt = { tab.data() };
		for (uint64_t u = 0; u < g.nunits; u++) st.flags |= qe_unit(qe_locate(g, u), cnt);
	}
	/* qe_table */
	int nt = im.ncomp > 1 ? 2 : 1;
	QeStd stdt = qe_std();
	for (int t = 0; t < 2 * nt; t++) {
		if (optimize) {
			std::vector<uint64_t> f(257); std::vector<int> cs(257), oth(257);
			qe_optimal(&tab[t], f.data(), cs.data(), oth.data(), 0, 1);
		} else qe_set_std(&tab[t], stdt, t);
		qe_codes(&tab[t]);
	}
	memcpy(out, head->prefix_dev, head->prefix_len);
	st.head_len = qe_header(im, g, tab.data(), out, cap);
	/* qe_len, qe_tscan (one scan over all units: the same offsets) */
	const uint32_t *csp[4] = { tab[0].cs, tab[1].cs, tab[2].cs, tab[3].cs };
	std::vector<uint64_t> off(g.nunits + 1, 0);
	for (uint64_t u = 0; u < g.nunits; u++) {
		QeLenSink s = { { csp[0], csp[1], csp[2], csp[3] }, 0 };
		st.flags |= qe_unit(qe_locate(g, u), s);
		off[u + 1] = off[u] + s.n;
	}
	st.total_bits = off[g.nunits]; st.nraw = (st.total_bits + 7) >> 3;
	/* qe_zero, qe_emit */
	std::vector<uint32_t> word((size_t)((st.total_bits + 31) / 32 + 1), 0);
	for (uint64_t u = 0; u < g.nunits; u++) qe_emit_unit(g, u, off[u], csp, word.data(), st.total_bits);
	/* qe_ffcount, qe_fscan, qe_copy */
	uint64_t pos = st.head_len;
	for (uint64_t c0 = 0; c0 < st.nraw; c0 += QE_CHUNK) {
		uint64_t c1 = c0 + QE_CHUNK < st.nraw ? c0 + QE_CHUNK : st.nraw;
		qe_stuff(word.data(), c0, c1, out, cap, pos);
		pos += (c1 - c0) + qe_ffs(word.data(), c0, c1);
	}
	uint64_t L = pos + 2;
	int32_t flags = (int32_t)st.flags;
	if (L > cap) flags |= JPEGQS_ENCODE_OVERFLOW;
	else { out[pos] = 0xFF; out[pos + 1] = 0xD9; }
	*len = L; *status = flags;
	return 0;
}

/* ================================================================ progressive mode (DESIGN.md section 3.14)
 * The file libjpeg writes for the same coefficients after jpeg_simple_progression with optimal tables
 * (progressive mode forces them): SOF2, then per scan [DHT ...] SOS data, each scan's data byte-aligned
 * with 1-bits and stuffed on its own.  Only compress_async reaches it.
 *
 *   unit      (scan, block) in scan order: interleaved MCU order for the DC scans, raster order over the
 *             component's real blocks for the AC scans.  Each scan's units start at a multiple of QE_T,
 *             so a tile of units belongs to one scan.
 *   padding   jccoefct.c compress_first_pass gives an MCU padding block the DC of its source (right
 *             edge: the last real block of its row; bottom rows: block h_samp - 1 of their MCU in the row
 *             above).  For the factors compress_async writes that is the last real block of its
 *             component before it in MCU order, qe_locate's predictor: a DC first difference of 0 and,
 *             in the DC refinement, bit Al of the source's DC.
 *   runs      an AC unit's symbols are local; the EOBn symbol of a run of blocks is given to the run's
 *             first block (after its own symbols) and every block of the run emits its own trailing
 *             correction bits after it - jcphuff.c's order.  Blocks that emit a symbol split a scan into
 *             segments; inside one, runs end at 0x7FFF blocks or when the correction bits exceed 937
 *             (MAX_CORR_BITS - DCTSIZE2 + 1).  qp_class scans (segment breaks, correction bits) per unit,
 *             qp_tscan per scan, and qp_runs walks each segment from its first block run by run,
 *             finding each run's end by a galloping search over those prefix sums.
 *   tables    qp_count gathers per-scan histograms, qp_table builds one optimal table per (scan, table
 *             used) with qe_optimal; then qp_len / qp_tscan / qp_emit / qp_ffcount / qp_fscan / qp_copy
 *             as the sequential passes, each scan's raw bytes starting on a chunk of their own.  qp_fscan
 *             places every scan and writes its DHT / SOS between the stuffed segments.
 */
#define QP_MAX_SCANS 10
#define QP_FIXED 73728                 /* descriptor + state + two tables per scan               */
#define QP_BLOCK_BITS 3928ull          /* a block's bits over all ten scans at most (DESIGN 3.14)  */
#define QP_HEAD_MAX 6000ull            /* DQT, SOF2, per scan DHT x 2 and SOS, EOI at most        */
#define QP_RUN_MAX 0x7FFFu             /* EOBRUN at which libjpeg flushes                         */
#define QP_BE_MAX 937u                 /* correction bits beyond which libjpeg flushes            */

struct QpScan {
	uint8_t ncomp, comp, ss, se, ah, al, pad[2];   /* comp: the AC scan's component                 */
	uint64_t n, ubase;                             /* units; the first (a multiple of QE_T)         */
};
struct QpScanState {
	uint64_t total;                    /* tile-scan total: (breaks << 32 | correction bits), then bits */
	uint64_t nraw, chunk0, data;       /* entropy-coded bytes; first chunk; file offset of the data   */
	uint32_t head, pad;                /* bytes of the scan's DHT / SOS                               */
};
struct QpState {
	uint64_t head_len, nchunk, len;    /* prefix + DQT + SOF2; chunks; file length                    */
	QpScanState sc[QP_MAX_SCANS];
};
struct QpImg {
	QeImg e;                           /* geometry 0, header fields, output, tab [2 per scan], ulen, tile, word, ffc */
	QpScan scan[QP_MAX_SCANS];
	int32_t nscan, pad;
	QpState *ps;
	uint8_t *cls;                      /* per unit: 1 ends in a run, 2 emits a symbol, correction bits << 2 */
	uint16_t *run;                     /* per unit: the run it starts, 0 for none                     */
	uint64_t *pre;                     /* per unit: (breaks << 32 | correction bits) before it in its tile */
};
static_assert(sizeof(QpImg) <= 2048 && sizeof(QpState) <= 2048 && 4096 + 2 * QP_MAX_SCANS * sizeof(QeTab) <= QP_FIXED, "qp fixed part");

/* jpeg_simple_progression's scripts for YCbCr and for one component */
static void qp_script(QpImg *p) {
	static const uint8_t col[QP_MAX_SCANS][5] = {      /* component (3: all), Ss, Se, Ah, Al */
		{ 3, 0, 0, 0, 1 }, { 0, 1, 5, 0, 2 }, { 2, 1, 63, 0, 1 }, { 1, 1, 63, 0, 1 }, { 0, 6, 63, 0, 2 },
		{ 0, 1, 63, 2, 1 }, { 3, 0, 0, 1, 0 }, { 2, 1, 63, 1, 0 }, { 1, 1, 63, 1, 0 }, { 0, 1, 63, 1, 0 } };
	static const uint8_t grey[6][5] = {
		{ 3, 0, 0, 0, 1 }, { 0, 1, 5, 0, 2 }, { 0, 6, 63, 0, 2 }, { 0, 1, 63, 2, 1 }, { 3, 0, 0, 1, 0 }, { 0, 1, 63, 1, 0 } };
	const QeGeo &g = p->e.geo[0];
	const bool colour = p->e.ncomp > 1;
	p->nscan = colour ? 10 : 6;
	uint64_t base = 0;
	for (int s = 0; s < p->nscan; s++) {
		const uint8_t *r = colour ? col[s] : grey[s];
		QpScan &sc = p->scan[s];
		memset(&sc, 0, sizeof(sc));
		sc.ncomp = r[0] == 3 ? (uint8_t)p->e.ncomp : 1; sc.comp = r[0] == 3 ? 0 : r[0];
		sc.ss = r[1]; sc.se = r[2]; sc.ah = r[3]; sc.al = r[4];
		sc.n = sc.ss == 0 ? g.nunits : (uint64_t)g.wblk[sc.comp] * g.hblk[sc.comp];
		sc.ubase = base;
		base += (sc.n + QE_T - 1) / QE_T * QE_T;
	}
}

/* table slots a scan uses: DC first 1 per DC table, DC refinement none, AC 1 */
HD static inline int qp_slots(const QpImg &p, const QpScan &sc) {
	return sc.ss ? 1 : sc.ah ? 0 : p.e.ncomp > 1 ? 2 : 1;
}

HD static inline int qp_scan_of(const QpImg &p, uint64_t u) {
	int s = 0;
	while (s + 1 < p.nscan && u >= p.scan[s + 1].ubase) s++;
	return s;
}

struct QpNull { HD void sym(int, int, uint32_t, int) {} HD void bits(uint32_t, int) {} };

/* n <= 63 buffered correction bits, the first the highest */
template <class S> HD static inline void qp_corr(S &sink, uint64_t b, int n) {
	if (n > 32) { sink.bits((uint32_t)(b >> 32), n - 32); n = 32; }
	if (n) sink.bits((uint32_t)b & (0xFFFFFFFFu >> (32 - n)), n);
}

/* emit_eobrun's symbol for a run of `run` blocks: EOBn, n = floor(log2 run), and the low n bits */
template <class S> HD static inline void qp_eobrun(S &sink, uint32_t run) {
	const int nb = qe_size((int)run) - 1;
	sink.sym(0, nb << 4, run & ((1u << nb) - 1), nb);
}

/* Unit i of scan sc, to sink.sym(slot, symbol, value bits, size) / sink.bits(bits, count), with `run`
 * the EOB run the unit starts (0 for none).  Returns its class: 1 it ends in an EOB run (jcphuff.c's
 * EOBRUN++), 2 it emits a symbol (so the pending run is flushed before it), and its trailing correction
 * bits << 2. */
template <class S> HD static inline uint32_t qp_unit(const QpImg &p, const QpScan &sc, uint64_t i, uint32_t run, S &sink) {
	const QeGeo &g = p.e.geo[0];
	const int al = sc.al;
	if (sc.ss == 0) {                                /* encode_mcu_DC_first / _refine */
		QeUnit un = qe_locate(g, i);
		const int dc = un.blk ? un.blk[0] : un.pred;
		if (sc.ah == 0) {
			const int diff = (dc >> al) - (un.pred >> al), s = qe_size(diff);
			sink.sym(un.tsel, s, (uint32_t)(diff + (diff >> 31)) & ((1u << s) - 1), s);
		} else sink.bits((uint32_t)(dc >> al) & 1u, 1);
		return 0;
	}
	const int16_t *blk = g.coef[sc.comp] + i * 64;
	uint64_t m = qe_zmask(blk) & ((~0ull << sc.ss) & (~0ull >> (63 - sc.se)));
	int prev = sc.ss - 1;
	if (sc.ah == 0) {                                /* encode_mcu_AC_first */
		uint32_t emits = 0;
		while (m) {
			const int k = qe_ctz64(m);
			m &= m - 1;
			const int v = blk[qe_nat(k)], a = (v < 0 ? -v : v) >> al;
			if (!a) continue;
			int r = k - prev - 1;
			prev = k; emits = 2;
			for (; r > 15; r -= 16) sink.sym(0, 0xF0, 0, 0);
			const int nb = qe_size(a);
			sink.sym(0, r << 4 | nb, (uint32_t)(v < 0 ? ~a : a) & ((1u << nb) - 1), nb);
		}
		if (run) qp_eobrun(sink, run);
		return (prev != sc.se ? 1u : 0u) | emits;
	}
	int eob = -1;                                    /* encode_mcu_AC_refine: the last newly-nonzero */
	for (uint64_t mm = m; mm; mm &= mm - 1) {
		const int k = qe_ctz64(mm), v = blk[qe_nat(k)];
		if (((v < 0 ? -v : v) >> al) == 1) eob = k;
	}
	int r = 0, nbr = 0;
	uint64_t br = 0;
	while (m) {
		const int k = qe_ctz64(m);
		m &= m - 1;
		const int v = blk[qe_nat(k)], a = (v < 0 ? -v : v) >> al;
		if (!a) continue;
		r += k - prev - 1;
		prev = k;
		while (r > 15 && k <= eob) { sink.sym(0, 0xF0, 0, 0); r -= 16; qp_corr(sink, br, nbr); br = 0; nbr = 0; }
		if (a > 1) { br = br << 1 | (uint64_t)(a & 1); nbr++; continue; }
		sink.sym(0, r << 4 | 1, v < 0 ? 0u : 1u, 1);
		qp_corr(sink, br, nbr); br = 0; nbr = 0; r = 0;
	}
	r += sc.se - prev;
	if (run) qp_eobrun(sink, run);
	qp_corr(sink, br, nbr);
	return (r > 0 || nbr > 0 ? 1u : 0u) | (eob >= 0 ? 2u : 0u) | (uint32_t)nbr << 2;
}

/* a unit that breaks its scan's runs: not in a run, the scan's first, one that emits a symbol, or one
 * after a unit not in a run.  Such a unit in a run starts a segment. */
HD static inline bool qp_break(uint32_t c, uint32_t cprev, uint64_t i) {
	return !(c & 1) || i == 0 || (c & 2) || !(cprev & 1);
}

/* (breaks << 32 | correction bits) of units [0, m) of scan s */
HD static inline uint64_t qp_pre(const QpImg &p, int s, uint64_t m) {
	const QpScan &sc = p.scan[s];
	if (m >= sc.n) return p.ps->sc[s].total;
	const uint64_t u = sc.ubase + m;
	return p.pre[u] + p.e.tile[u / QE_T];
}

/* the smallest m in [lo, hi] with field(P(m)) - base > lim (monotone in m), hi + 1 if none: a gallop
 * from lo, then bisection */
HD static inline uint64_t qp_first(const QpImg &p, int s, bool high, uint64_t base, uint64_t lim, uint64_t lo, uint64_t hi) {
	uint64_t a = lo, b = lo, step = 1;
	for (;;) {
		if (b > hi) return hi + 1;
		const uint64_t v = qp_pre(p, s, b), x = high ? v >> 32 : v & 0xFFFFFFFFull;
		if (x - base > lim) break;
		a = b + 1;
		if (b == hi) return hi + 1;
		b = b + step > hi ? hi : b + step;
		step <<= 1;
	}
	while (a < b) {
		const uint64_t mid = a + (b - a) / 2, v = qp_pre(p, s, mid), x = high ? v >> 32 : v & 0xFFFFFFFFull;
		if (x - base > lim) b = mid; else a = mid + 1;
	}
	return a;
}

/* the runs of the segment starting at unit j of scan s: each starts with EOBRUN 0 and BE 0 and ends
 * after QP_RUN_MAX blocks, after the block that takes BE past QP_BE_MAX, or at the segment's end */
HD static inline void qp_walk(const QpImg &p, int s, uint64_t j) {
	const QpScan &sc = p.scan[s];
	const uint64_t pj = qp_pre(p, s, j);
	const uint64_t end = qp_first(p, s, true, pj >> 32, 1, j + 2, sc.n) - 1;   /* the next break, or n */
	for (uint64_t r = j; r < end;) {
		const uint64_t pr = r == j ? pj : qp_pre(p, s, r);
		const uint64_t lim = r + QP_RUN_MAX < end ? r + QP_RUN_MAX : end;
		uint64_t e = qp_first(p, s, false, pr & 0xFFFFFFFFull, QP_BE_MAX, r + 1, lim);
		if (e > lim) e = lim;
		p.run[sc.ubase + r] = (uint16_t)(e - r);
		r = e;
	}
}

/* the scan's DHT for every table it uses, then its SOS (jcmarker.c write_scan_header) */
HD static inline void qp_scan_head(const QpImg &p, int s, const QeTab *tab, QeOut &o) {
	const QpScan &sc = p.scan[s];
	for (int t = 0; t < qp_slots(p, sc); t++) {
		const QeTab &h = tab[2 * s + t];
		const int id = sc.ss ? (sc.comp ? 1 : 0) : t;
		o.w(0xFFC4); o.w(2 + 1 + 16 + h.nval); o.b((unsigned)((sc.ss ? 0x10 : 0) | id));
		for (int l = 1; l <= 16; l++) o.b(h.bits[l]);
		for (int l = 0; l < h.nval; l++) o.b(h.val[l]);
	}
	o.w(0xFFDA); o.w(6 + 2 * sc.ncomp); o.b(sc.ncomp);
	for (int k = 0; k < sc.ncomp; k++) {
		const int c = sc.ncomp > 1 ? k : sc.comp;
		const unsigned td = sc.ss == 0 && sc.ah == 0 && c ? 1 : 0, ta = sc.se && c ? 1 : 0;
		o.b((unsigned)p.e.comp_id[c]); o.b(td << 4 | ta);
	}
	o.b(sc.ss); o.b(sc.se); o.b((unsigned)(sc.ah << 4 | sc.al));
}

struct QpLenSink {
	const uint32_t *cs[2]; uint32_t n;
	HD void sym(int t, int s, uint32_t, int nv) { n += (cs[t][s] & 255) + (uint32_t)nv; }
	HD void bits(uint32_t, int nv) { n += (uint32_t)nv; }
};
struct QpEmitSink {
	const uint32_t *cs[2]; QeEmitSink e;
	HD void sym(int t, int s, uint32_t vb, int nv) { const uint32_t c = cs[t][s]; e.put((c >> 8) << nv | vb, (int)(c & 255) + nv); }
	HD void bits(uint32_t v, int nv) { e.put(v, nv); }
};

/* unit i of scan s written from bit offset o on; the scan's last unit pads its byte with 1-bits */
HD static inline void qp_emit_unit(const QpImg &p, int s, uint64_t i, uint32_t run, uint64_t o, const uint32_t *cs0,
		const uint32_t *cs1, uint64_t total) {
	QpEmitSink k;
	k.cs[0] = cs0; k.cs[1] = cs1;
	k.e.w = p.e.word; k.e.base = o & ~31ull; k.e.acc = 0; k.e.nacc = (int)(o & 31); k.e.shared = (o & 31) != 0;
	qp_unit(p, p.scan[s], i, run, k);
	if (i + 1 == p.scan[s].n) {
		const int pad = (int)((8 - (total & 7)) & 7);
		if (pad) k.e.put((1u << pad) - 1, pad);
	}
	k.e.finish();
}

/* the scan a chunk of raw bytes belongs to, -1 for none */
HD static inline int qp_chunk_scan(const QpImg &p, uint64_t c) {
	for (int s = 0; s < p.nscan; s++) {
		const QpScanState &t = p.ps->sc[s];
		if (c >= t.chunk0 && c < t.chunk0 + (t.nraw + QE_CHUNK - 1) / QE_CHUNK) return s;
	}
	return -1;
}

/* ---------------------------------------------------------------- progressive kernels */
struct QpSetupPack { QpImg img[QE_PACK]; int n; };
static_assert(sizeof(QpSetupPack) <= 32000, "QpSetupPack exceeds the kernel parameter space");
struct QpPtrs { const QpImg *img[QE_PACK]; int n; };

__global__ void __launch_bounds__(256) qp_setup_kernel(const __grid_constant__ QpSetupPack P) {
	const int i = blockIdx.x;
	if (i >= P.n) return;
	const QpImg &p = P.img[i];
	if (threadIdx.x == 0) {
		*reinterpret_cast<QpImg *>(reinterpret_cast<char *>(p.ps) - 2048) = p;
		memset(p.ps, 0, sizeof(QpState));
	}
	for (int j = threadIdx.x; j < 2 * p.nscan * 257; j += blockDim.x) p.e.tab[j / 257].freq[j % 257] = 0;
}

/* per tile: every unit's class and run slot; the in-tile exclusive scan of (break << 32 | correction
 * bits); the tile's sum */
__global__ void __launch_bounds__(QE_T) qp_class_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QpImg &p = *P.img[blockIdx.y];
	const uint64_t u0 = (uint64_t)blockIdx.x * QE_T;
	if (u0 >= p.scan[p.nscan - 1].ubase + p.scan[p.nscan - 1].n) return;
	const int s = qp_scan_of(p, u0);
	const QpScan &sc = p.scan[s];
	const uint64_t u = u0 + threadIdx.x, i = u - sc.ubase;
	__shared__ uint8_t s_cls[QE_T];
	QpNull z;
	uint32_t c = 0;
	if (i < sc.n) {
		if (sc.ss) c = qp_unit(p, sc, i, 0, z);
		p.cls[u] = (uint8_t)c; p.run[u] = 0;
	}
	s_cls[threadIdx.x] = (uint8_t)c;
	__syncthreads();
	uint64_t v = 0;
	if (i < sc.n && sc.ss) {
		uint32_t cp = 0;
		if (i > 0) cp = threadIdx.x ? s_cls[threadIdx.x - 1] : qp_unit(p, sc, i - 1, 0, z);
		v = (qp_break(c, cp, i) ? 1ull << 32 : 0) | (c >> 2);
	}
	typedef cub::BlockScan<uint64_t, QE_T> S;
	__shared__ typename S::TempStorage tmp;
	uint64_t ex, agg;
	S(tmp).ExclusiveSum(v, ex, agg);
	if (i < sc.n) p.pre[u] = ex;
	if (threadIdx.x == 0) p.e.tile[blockIdx.x] = agg;
}

/* per image: the tile sums scanned per scan (exclusive, restarting at every scan) and each scan's total;
 * with `bits`, also each scan's raw bytes and first chunk */
__global__ void __launch_bounds__(QE_SCAN_T) qp_tscan_kernel(const __grid_constant__ QpPtrs P, int bits) {
	if ((int)blockIdx.x >= P.n) return;
	const QpImg &p = *P.img[blockIdx.x];
	typedef cub::BlockScan<uint64_t, QE_SCAN_T> S;
	__shared__ typename S::TempStorage tmp;
	for (int s = 0; s < p.nscan; s++) {
		const QpScan &sc = p.scan[s];
		const uint64_t t0 = sc.ubase / QE_T, nt = (sc.n + QE_T - 1) / QE_T;
		uint64_t carry = 0;
		for (uint64_t base = 0; base < nt; base += QE_SCAN_T) {
			const uint64_t t = base + threadIdx.x;
			uint64_t v = t < nt ? p.e.tile[t0 + t] : 0, ex, agg;
			S(tmp).ExclusiveSum(v, ex, agg);
			if (t < nt) p.e.tile[t0 + t] = carry + ex;
			carry += agg;
			__syncthreads();
		}
		if (threadIdx.x == 0) p.ps->sc[s].total = carry;
	}
	if (bits && threadIdx.x == 0) {
		uint64_t c = 0;
		for (int s = 0; s < p.nscan; s++) {
			QpScanState &t = p.ps->sc[s];
			t.nraw = (t.total + 7) >> 3; t.chunk0 = c;
			c += (t.nraw + QE_CHUNK - 1) / QE_CHUNK;
		}
		p.ps->nchunk = c;
	}
}

/* per unit: the segments of the AC scans walked from their first units */
__global__ void __launch_bounds__(QE_T) qp_runs_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QpImg &p = *P.img[blockIdx.y];
	const uint64_t u0 = (uint64_t)blockIdx.x * QE_T;
	if (u0 >= p.scan[p.nscan - 1].ubase + p.scan[p.nscan - 1].n) return;
	const int s = qp_scan_of(p, u0);
	const QpScan &sc = p.scan[s];
	const uint64_t u = u0 + threadIdx.x, i = u - sc.ubase;
	if (!sc.ss || i >= sc.n) return;
	const uint32_t c = p.cls[u];
	if ((c & 1) && qp_break(c, i ? p.cls[u - 1] : 0, i)) qp_walk(p, s, i);
}

struct QpCountSink {
	uint32_t (*h)[257];
	__device__ void sym(int t, int s, uint32_t, int) { atomicAdd(&h[t][s], 1u); }
	__device__ void bits(uint32_t, int) {}
};

/* per tile: its units' symbols into shared histograms, then into the scan's tables */
__global__ void __launch_bounds__(QE_T) qp_count_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QpImg &p = *P.img[blockIdx.y];
	const uint64_t u0 = (uint64_t)blockIdx.x * QE_T;
	if (u0 >= p.scan[p.nscan - 1].ubase + p.scan[p.nscan - 1].n) return;
	const int s = qp_scan_of(p, u0);
	const QpScan &sc = p.scan[s];
	if (sc.ss == 0 && sc.ah) return;                 /* the DC refinement codes no symbol */
	__shared__ uint32_t h[2][257];
	for (int j = threadIdx.x; j < 2 * 257; j += QE_T) h[j / 257][j % 257] = 0;
	__syncthreads();
	const uint64_t u = u0 + threadIdx.x, i = u - sc.ubase;
	if (i < sc.n) { QpCountSink k = { h }; qp_unit(p, sc, i, p.run[u], k); }
	__syncthreads();
	for (int j = threadIdx.x; j < 2 * 257; j += QE_T) {
		const uint32_t v = h[j / 257][j % 257];
		if (v) atomicAdd(reinterpret_cast<unsigned long long *>(&p.e.tab[2 * s + j / 257].freq[j % 257]), (unsigned long long)v);
	}
}

/* blockIdx = (scan, image), warp w = the scan's table w: the optimal table and its codes; the scan's
 * DHT / SOS length; scan 0 also copies the prefix and writes DQT and SOF2 */
__global__ void __launch_bounds__(64) qp_table_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QpImg &p = *P.img[blockIdx.y];
	const int s = blockIdx.x;
	if (s >= p.nscan) return;
	__shared__ uint64_t s_freq[2][257];
	__shared__ int s_size[2][257], s_oth[2][257];
	const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
	if (w < qp_slots(p, p.scan[s])) {
		QeTab *t = p.e.tab + 2 * s + w;
		qe_optimal(t, s_freq[w], s_size[w], s_oth[w], lane, 32);
		if (lane == 0) qe_codes(t);
	}
	if (s == 0) for (uint64_t j = threadIdx.x; j < p.e.prefix_len && j < p.e.cap; j += blockDim.x) p.e.out[j] = p.e.prefix[j];
	__syncthreads();
	if (threadIdx.x == 0) {
		QeOut o = { NULL, 0, 0 };
		qp_scan_head(p, s, p.e.tab, o);
		p.ps->sc[s].head = (uint32_t)o.n;
		if (s == 0) {
			QeOut f = { p.e.out, p.e.cap, p.e.prefix_len };
			qe_frame(p.e, p.e.geo[0], f, true);
			p.ps->head_len = f.n;
		}
	}
}

/* per tile: every unit's bit length with its scan's tables, the tile's sum */
__global__ void __launch_bounds__(QE_T) qp_len_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QpImg &p = *P.img[blockIdx.y];
	const uint64_t u0 = (uint64_t)blockIdx.x * QE_T;
	if (u0 >= p.scan[p.nscan - 1].ubase + p.scan[p.nscan - 1].n) return;
	const int s = qp_scan_of(p, u0);
	const QpScan &sc = p.scan[s];
	__shared__ uint32_t s_cs[2][256];
	for (int j = threadIdx.x; j < 2 * 256; j += QE_T) s_cs[j >> 8][j & 255] = p.e.tab[2 * s + (j >> 8)].cs[j & 255];
	__syncthreads();
	const uint64_t u = u0 + threadIdx.x, i = u - sc.ubase;
	uint32_t n = 0;
	if (i < sc.n) {
		QpLenSink k = { { s_cs[0], s_cs[1] }, 0 };
		qp_unit(p, sc, i, p.run[u], k);
		n = k.n;
		p.e.ulen[u] = (uint16_t)n;
	}
	typedef cub::BlockReduce<uint32_t, QE_T> R;
	__shared__ typename R::TempStorage tmp;
	const uint32_t sum = R(tmp).Sum(n);
	if (threadIdx.x == 0) p.e.tile[blockIdx.x] = sum;
}

/* the words every scan's bits will occupy, and one more, set to zero */
__global__ void __launch_bounds__(256) qp_zero_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QpImg &p = *P.img[blockIdx.y];
	const uint64_t nw = p.ps->nchunk * (QE_CHUNK / 4) + 1;
	for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nw; j += (uint64_t)gridDim.x * blockDim.x) p.e.word[j] = 0;
}

/* per tile: the units' bit offsets (scan's first chunk + tile offset + scan inside the tile), their bits */
__global__ void __launch_bounds__(QE_T) qp_emit_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QpImg &p = *P.img[blockIdx.y];
	const uint64_t u0 = (uint64_t)blockIdx.x * QE_T;
	if (u0 >= p.scan[p.nscan - 1].ubase + p.scan[p.nscan - 1].n) return;
	const int s = qp_scan_of(p, u0);
	const QpScan &sc = p.scan[s];
	__shared__ uint32_t s_cs[2][256];
	for (int j = threadIdx.x; j < 2 * 256; j += QE_T) s_cs[j >> 8][j & 255] = p.e.tab[2 * s + (j >> 8)].cs[j & 255];
	const uint64_t u = u0 + threadIdx.x, i = u - sc.ubase;
	const uint32_t n = i < sc.n ? p.e.ulen[u] : 0;
	uint32_t ex;
	typedef cub::BlockScan<uint32_t, QE_T> S;
	__shared__ typename S::TempStorage tmp;
	S(tmp).ExclusiveSum(n, ex);
	__syncthreads();
	if (i < sc.n) {
		const QpScanState &t = p.ps->sc[s];
		qp_emit_unit(p, s, i, p.run[u], t.chunk0 * QE_CHUNK * 8 + p.e.tile[blockIdx.x] + ex, s_cs[0], s_cs[1], t.total);
	}
}

/* per chunk of a scan's raw bytes: its 0xFF bytes */
__global__ void __launch_bounds__(QE_BT) qp_ffcount_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QpImg &p = *P.img[blockIdx.y];
	const uint64_t c = blockIdx.x;
	if (c >= p.ps->nchunk) return;
	const int s = qp_chunk_scan(p, c);
	const uint64_t end = s < 0 ? 0 : p.ps->sc[s].chunk0 * QE_CHUNK + p.ps->sc[s].nraw;
	const uint64_t j0 = c * QE_CHUNK + threadIdx.x * 16, j1 = j0 + 16 < end ? j0 + 16 : end;
	const uint32_t n = j0 < end ? qe_ffs(p.e.word, j0, j1) : 0;
	typedef cub::BlockReduce<uint32_t, QE_BT> R;
	__shared__ typename R::TempStorage tmp;
	const uint32_t sum = R(tmp).Sum(n);
	if (threadIdx.x == 0) p.e.ffc[c] = sum;
}

/* per image: exclusive scan of the chunk counts; every scan's place in the file and its DHT / SOS; file
 * length, status, EOI */
__global__ void __launch_bounds__(QE_SCAN_T) qp_fscan_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.x >= P.n) return;
	const QpImg &p = *P.img[blockIdx.x];
	QpState *ps = p.ps;
	const uint64_t nchunk = ps->nchunk;
	uint64_t carry = 0;
	typedef cub::BlockScan<uint64_t, QE_SCAN_T> S;
	__shared__ typename S::TempStorage tmp;
	for (uint64_t base = 0; base < nchunk; base += QE_SCAN_T) {
		const uint64_t c = base + threadIdx.x;
		uint64_t v = c < nchunk ? p.e.ffc[c] : 0, ex, agg;
		S(tmp).ExclusiveSum(v, ex, agg);
		if (c < nchunk) p.e.ffc[c] = (uint32_t)(carry + ex);
		carry += agg;
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		uint64_t pos = ps->head_len;
		for (int s = 0; s < p.nscan; s++) {
			QpScanState &t = ps->sc[s];
			const uint64_t c1 = t.chunk0 + (t.nraw + QE_CHUNK - 1) / QE_CHUNK;
			const uint64_t ff = (c1 < nchunk ? p.e.ffc[c1] : carry) - (t.chunk0 < nchunk ? p.e.ffc[t.chunk0] : carry);
			t.data = pos + t.head;
			pos = t.data + t.nraw + ff;
		}
		const uint64_t L = pos + 2;
		int32_t flags = 0;
		if (L > p.e.cap) flags |= JPEGQS_ENCODE_OVERFLOW;
		else { p.e.out[pos] = 0xFF; p.e.out[pos + 1] = 0xD9; }
		ps->len = L;
		*p.e.len = L;
		*p.e.status = flags;
	}
	__syncthreads();
	const int w = threadIdx.x >> 5;
	if (w < p.nscan && (threadIdx.x & 31) == 0) {
		QeOut o = { p.e.out, p.e.cap, ps->sc[w].data - ps->sc[w].head };
		qp_scan_head(p, w, p.e.tab, o);
	}
}

/* per chunk: its bytes stuffed to the output */
__global__ void __launch_bounds__(QE_BT) qp_copy_kernel(const __grid_constant__ QpPtrs P) {
	if ((int)blockIdx.y >= P.n) return;
	const QpImg &p = *P.img[blockIdx.y];
	const uint64_t c = blockIdx.x;
	if (c >= p.ps->nchunk) return;
	const int s = qp_chunk_scan(p, c);
	if (s < 0) return;
	const QpScanState &t = p.ps->sc[s];
	const uint64_t b0 = t.chunk0 * QE_CHUNK, end = b0 + t.nraw;
	const uint64_t j0 = c * QE_CHUNK + threadIdx.x * 16, j1 = j0 + 16 < end ? j0 + 16 : end;
	uint32_t n = j0 < end ? qe_ffs(p.e.word, j0, j1) : 0, ex;
	typedef cub::BlockScan<uint32_t, QE_BT> S;
	__shared__ typename S::TempStorage tmp;
	S(tmp).ExclusiveSum(n, ex);
	if (j0 < end) qe_stuff(p.e.word, j0, j1, p.e.out, p.e.cap, t.data + (j0 - b0) + (p.e.ffc[c] - p.e.ffc[t.chunk0]) + ex);
}

/* ---------------------------------------------------------------- progressive host side */
struct QpSizes { uint64_t units, tiles, words, chunks; size_t bytes; };

/* the workspace of an image: units of the ten (six) scans, each rounded up to QE_T; raw words for
 * U * QP_BLOCK_BITS bits plus a chunk of alignment per scan */
static QpSizes qp_sizes(const QpImg &p) {
	QpSizes z;
	const QpScan &last = p.scan[p.nscan - 1];
	z.units = last.ubase + (last.n + QE_T - 1) / QE_T * QE_T;
	z.tiles = z.units / QE_T;
	z.words = (p.e.geo[0].nunits * QP_BLOCK_BITS + 31) / 32 + QP_MAX_SCANS * (QE_CHUNK / 4) + 2;
	z.chunks = (4 * z.words + QE_CHUNK - 1) / QE_CHUNK;
	z.bytes = QP_FIXED + qe_a256(z.units) + qe_a256(2 * z.units) + qe_a256(8 * z.units) + qe_a256(2 * z.units) +
		qe_a256(8 * z.tiles) + qe_a256(4 * z.words) + qe_a256(4 * z.chunks);
	return z;
}

static void qp_carve(QpImg *p, const QpSizes &z, char *w) {
	p->ps = reinterpret_cast<QpState *>(w + 2048);
	p->e.tab = reinterpret_cast<QeTab *>(w + 4096);
	w += QP_FIXED;
	p->cls = reinterpret_cast<uint8_t *>(w); w += qe_a256(z.units);
	p->run = reinterpret_cast<uint16_t *>(w); w += qe_a256(2 * z.units);
	p->pre = reinterpret_cast<uint64_t *>(w); w += qe_a256(8 * z.units);
	p->e.ulen = reinterpret_cast<uint16_t *>(w); w += qe_a256(2 * z.units);
	p->e.tile = reinterpret_cast<uint64_t *>(w); w += qe_a256(8 * z.tiles);
	p->e.word = reinterpret_cast<uint32_t *>(w); w += qe_a256(4 * z.words);
	p->e.ffc = reinterpret_cast<uint32_t *>(w);
}

/* checks image i with its head and fills its descriptor (no workspace yet) */
static const char *qp_check(const jpegqs_cuda_image *im, const jpegqs_cuda_jpeg_head *hd, QpImg *p, QpSizes *z) {
	memset(p, 0, sizeof(*p));
	QeSizes unused;
	const char *e = qe_check(im, hd, false, 1, &p->e, &unused);
	if (e) return e;
	if (p->e.upmode) return "progressive mode codes the sampled geometry only";
	if (im->ncomp != 1 && im->ncomp != 3) return "progressive mode takes 1 or 3 components";
	qp_script(p);
	*z = qp_sizes(*p);
	return NULL;
}

/* the progressive file's bound and workspace for an image compress_async makes */
size_t qe_progressive_bound(const jpegqs_cuda_image *img, size_t prefix_len) {
	QeGeo g0, g1; bool up;
	if (qe_geometry(img, &g0, &g1, &up)) return 0;
	return prefix_len + QP_HEAD_MAX + 2 * ((g0.nunits * QP_BLOCK_BITS + 7) / 8 + QP_MAX_SCANS);
}
size_t qe_progressive_workspace(const jpegqs_cuda_image *img) {
	QpImg p;
	memset(&p, 0, sizeof(p));
	QeGeo g1; bool up;
	if (qe_geometry(img, &p.e.geo[0], &g1, &up)) return 0;
	p.e.ncomp = img->ncomp;
	qp_script(&p);
	return qp_sizes(p).bytes;
}

/* the progressive encoder over device coefficients, as encode_async's stream rules; launches as
 * qs_ctx_decode_done records them */
int qe_progressive_async(jpegqs_cuda_ctx *ctx, int n, const jpegqs_cuda_image *imgs, const jpegqs_cuda_jpeg_head *heads,
		uint8_t *const *out_dev, const size_t *out_cap, uint64_t *len_dev, int32_t *status_dev, void *workspace,
		size_t workspace_bytes, cudaStream_t st) {
	char msg[512] = "";
	int launches = 0;
	std::vector<QpImg> desc((size_t)n);
	std::vector<QpSizes> sizes((size_t)n);
	size_t need = 0;
	for (int i = 0; i < n; i++) {
		const char *e = qp_check(&imgs[i], &heads[i], &desc[i], &sizes[i]);
		if (e) { snprintf(msg, sizeof(msg), "progressive encoder: image %d: %s", i, e); qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG; }
		need += sizes[i].bytes;
	}
	if (workspace_bytes < need || ((uintptr_t)workspace & 255)) {
		snprintf(msg, sizeof(msg), "progressive encoder: workspace of %zu bytes, %zu needed", workspace_bytes, need);
		qs_ctx_decode_done(ctx, 0, msg); return JPEGQS_ERR_ARG;
	}
	char *w = (char *)workspace;
	for (int i = 0; i < n; i++) {
		QpImg &d = desc[i];
		qp_carve(&d, sizes[i], w); w += sizes[i].bytes;
		d.e.index = i; d.e.out = out_dev[i]; d.e.cap = out_cap[i]; d.e.len = len_dev + i; d.e.status = status_dev + i;
	}
	for (int g0 = 0; g0 < n; g0 += QE_PACK) {
		const int g = n - g0 < QE_PACK ? n - g0 : QE_PACK;
		std::unique_ptr<QpSetupPack> hold(new QpSetupPack());
		QpSetupPack &pack = *hold;
		QpPtrs P;
		memset(&pack, 0, sizeof(pack)); memset(&P, 0, sizeof(P));
		pack.n = g; P.n = g;
		uint64_t maxtile = 1, maxchunk = 1;
		for (int j = 0; j < g; j++) {
			pack.img[j] = desc[g0 + j];
			P.img[j] = reinterpret_cast<const QpImg *>(reinterpret_cast<const char *>(desc[g0 + j].ps) - 2048);
			if (sizes[g0 + j].tiles > maxtile) maxtile = sizes[g0 + j].tiles;
			if (sizes[g0 + j].chunks > maxchunk) maxchunk = sizes[g0 + j].chunks;
		}
		if (maxtile > 0x7FFFFFFFull || maxchunk > 0x7FFFFFFFull) { qs_ctx_decode_done(ctx, launches, "progressive encoder: image too large"); return JPEGQS_ERR_ARG; }
		const dim3 tiles((unsigned)maxtile, g), chunks((unsigned)maxchunk, g);
		const unsigned zero_blocks = (unsigned)(maxchunk < 4096 ? maxchunk : 4096);
		qp_setup_kernel<<<g, 256, 0, st>>>(pack); launches++;
		qp_class_kernel<<<tiles, QE_T, 0, st>>>(P); launches++;
		qp_tscan_kernel<<<g, QE_SCAN_T, 0, st>>>(P, 0); launches++;
		qp_runs_kernel<<<tiles, QE_T, 0, st>>>(P); launches++;
		qp_count_kernel<<<tiles, QE_T, 0, st>>>(P); launches++;
		qp_table_kernel<<<dim3(QP_MAX_SCANS, g), 64, 0, st>>>(P); launches++;
		qp_len_kernel<<<tiles, QE_T, 0, st>>>(P); launches++;
		qp_tscan_kernel<<<g, QE_SCAN_T, 0, st>>>(P, 1); launches++;
		qp_zero_kernel<<<dim3(zero_blocks, g), 256, 0, st>>>(P); launches++;
		qp_emit_kernel<<<tiles, QE_T, 0, st>>>(P); launches++;
		qp_ffcount_kernel<<<chunks, QE_BT, 0, st>>>(P); launches++;
		qp_fscan_kernel<<<g, QE_SCAN_T, 0, st>>>(P); launches++;
		qp_copy_kernel<<<chunks, QE_BT, 0, st>>>(P); launches++;
		QE_CK(cudaGetLastError());
	}
	qs_ctx_decode_done(ctx, launches, "");
	return 0;
}

/* the same steps on the calling thread: every per-unit function in the kernels' order, each scan's
 * prefix sums taken over the whole scan (tile offsets 0) */
int qe_progressive_model(const jpegqs_cuda_image *img, const jpegqs_cuda_jpeg_head *head, uint8_t *out, size_t cap,
		uint64_t *len, int32_t *status) {
	QpImg p; QpSizes z;
	const char *e = qp_check(img, head, &p, &z);
	if (!e && cap < head->prefix_len) e = "cap smaller than prefix_len";
	if (e) { char m[256]; snprintf(m, sizeof(m), "progressive model: %s", e); qs_set_host_error(m); return JPEGQS_ERR_ARG; }
	QpState ps;
	memset(&ps, 0, sizeof(ps));
	std::vector<QeTab> tab(2 * QP_MAX_SCANS);
	memset(tab.data(), 0, tab.size() * sizeof(QeTab));
	std::vector<uint8_t> cls(z.units, 0);
	std::vector<uint16_t> run(z.units, 0);
	std::vector<uint64_t> pre(z.units, 0), tile(z.tiles, 0);
	p.ps = &ps; p.e.tab = tab.data(); p.cls = cls.data(); p.run = run.data(); p.pre = pre.data(); p.e.tile = tile.data();
	p.e.out = out; p.e.cap = cap;
	QpNull zs;
	/* qp_class, qp_tscan, qp_runs */
	for (int s = 0; s < p.nscan; s++) {
		const QpScan &sc = p.scan[s];
		if (!sc.ss) continue;
		uint64_t acc = 0; uint32_t cp = 0;
		for (uint64_t i = 0; i < sc.n; i++) {
			const uint32_t c = qp_unit(p, sc, i, 0, zs);
			cls[sc.ubase + i] = (uint8_t)c;
			pre[sc.ubase + i] = acc;
			acc += (qp_break(c, cp, i) ? 1ull << 32 : 0) | (c >> 2);
			cp = c;
		}
		ps.sc[s].total = acc;
		for (uint64_t i = 0; i < sc.n; i++) {
			const uint32_t c = cls[sc.ubase + i];
			if ((c & 1) && qp_break(c, i ? cls[sc.ubase + i - 1] : 0, i)) qp_walk(p, s, i);
		}
	}
	/* qp_count, qp_table */
	for (int s = 0; s < p.nscan; s++) {
		const QpScan &sc = p.scan[s];
		struct { QeTab *t; void sym(int k, int v, uint32_t, int) { t[k].freq[v]++; } void bits(uint32_t, int) {} } cnt = { tab.data() + 2 * s };
		if (qp_slots(p, sc)) for (uint64_t i = 0; i < sc.n; i++) qp_unit(p, sc, i, run[sc.ubase + i], cnt);
		for (int t = 0; t < qp_slots(p, sc); t++) {
			std::vector<uint64_t> f(257); std::vector<int> cs(257), oth(257);
			qe_optimal(&tab[2 * s + t], f.data(), cs.data(), oth.data(), 0, 1);
			qe_codes(&tab[2 * s + t]);
		}
	}
	memcpy(out, head->prefix_dev, head->prefix_len);
	QeOut f = { out, cap, head->prefix_len };
	qe_frame(p.e, p.e.geo[0], f, true);
	/* qp_len, qp_emit per scan, then the stuffed copy between the scan headers */
	uint64_t pos = f.n;
	for (int s = 0; s < p.nscan; s++) {
		const QpScan &sc = p.scan[s];
		const uint32_t *cs0 = tab[2 * s].cs, *cs1 = tab[2 * s + 1].cs;
		std::vector<uint64_t> off(sc.n + 1, 0);
		for (uint64_t i = 0; i < sc.n; i++) {
			QpLenSink k = { { cs0, cs1 }, 0 };
			qp_unit(p, sc, i, run[sc.ubase + i], k);
			off[i + 1] = off[i] + k.n;
		}
		const uint64_t total = off[sc.n], nraw = (total + 7) >> 3;
		std::vector<uint32_t> word((size_t)((total + 31) / 32 + 1), 0);
		p.e.word = word.data();
		for (uint64_t i = 0; i < sc.n; i++) qp_emit_unit(p, s, i, run[sc.ubase + i], off[i], cs0, cs1, total);
		QeOut o = { out, cap, pos };
		qp_scan_head(p, s, tab.data(), o);
		pos = o.n;
		qe_stuff(word.data(), 0, nraw, out, cap, pos);
		pos += nraw + qe_ffs(word.data(), 0, nraw);
	}
	const uint64_t L = pos + 2;
	int32_t flags = 0;
	if (L > cap) flags |= JPEGQS_ENCODE_OVERFLOW;
	else { out[pos] = 0xFF; out[pos + 1] = 0xD9; }
	*len = L; *status = flags;
	return 0;
}
