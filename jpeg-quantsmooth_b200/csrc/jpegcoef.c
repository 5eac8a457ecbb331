/*
 * jpegcoef.c - JPEG coefficient reader / writer (see jpegcoef.h).  Written from ITU-T T.81:
 * marker syntax (Annex B), Huffman decoding (F.2.2), progressive procedures (G.1.2 / G.2),
 * Huffman table generation (C.2, K.2) and the example tables of K.3.  It stands in for the
 * jpeg_read_coefficients / jpeg_write_coefficients calls of the reference CLI
 * (reference quantsmooth.c:548-549, 579-596).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <time.h>
#include <pthread.h>
#include <unistd.h>
#ifdef __SSE2__
#include <emmintrin.h>
#endif
#include "jpegcoef.h"

/* for the JPEGQS_CODEC_TRACE=1 lines (which path ran, how long it took) */
static double trace_ms(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }

/* zig-zag index -> natural (row-major) index, T.81 figure A.6 */
static const unsigned char zz_nat[64 + 16] = {
	0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
	28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
	54, 47, 55, 62, 63,
	63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63       /* guard for corrupt run lengths */
};

/* Which coefficients of a block are not zero, as a bit mask in ZIG-ZAG order (bit k = k-th
 * coefficient of the scan): the block coder and the progressive refinement decoder walk the set
 * bits instead of testing 63 coefficients.  Natural-order mask by 16-bit compares (SSE2 when the
 * target has it), turned into zig-zag order with one table look-up per block row. */
static uint64_t zz_mask_tab[8][256];
static pthread_once_t zz_mask_once = PTHREAD_ONCE_INIT;
static void zz_mask_init(void) {
	int r, b, c, k; unsigned char nat_zz[64];
	for (k = 0; k < 64; k++) nat_zz[zz_nat[k]] = (unsigned char)k;
	for (r = 0; r < 8; r++) for (b = 0; b < 256; b++) {
		uint64_t m = 0;
		for (c = 0; c < 8; c++) if (b >> c & 1) m |= 1ULL << nat_zz[r * 8 + c];
		zz_mask_tab[r][b] = m;
	}
}
static inline uint64_t nonzero_mask_zz(const JCOEF *blk) {
	uint64_t m = 0; int r;
#ifdef __SSE2__
	const __m128i z = _mm_setzero_si128();
	for (r = 0; r < 8; r += 2) {
		__m128i a = _mm_cmpeq_epi16(_mm_loadu_si128((const __m128i*)(blk + r * 8)), z);
		__m128i b = _mm_cmpeq_epi16(_mm_loadu_si128((const __m128i*)(blk + r * 8 + 8)), z);
		unsigned k = ~(unsigned)_mm_movemask_epi8(_mm_packs_epi16(a, b));     /* bit set = coefficient not zero */
		m |= zz_mask_tab[r][k & 255] | zz_mask_tab[r + 1][k >> 8 & 255];
	}
#else
	for (r = 0; r < 8; r++) {
		unsigned k = 0; int c;
		for (c = 0; c < 8; c++) k |= (unsigned)(blk[r * 8 + c] != 0) << c;
		m |= zz_mask_tab[r][k];
	}
#endif
	return m;
}
/* The same for the AC coefficients only, WITHOUT reading blk[0]: a DC scan may be writing it on
 * another thread while a refinement scan of the AC band walks the block ("progressive scans side
 * by side" below). */
static inline uint64_t nonzero_mask_zz_ac(const JCOEF *blk) {
	uint64_t m = 0; int r;
#ifdef __SSE2__
	const __m128i z = _mm_setzero_si128();
	{
		__m128i a = _mm_cmpeq_epi16(_mm_slli_si128(_mm_loadu_si128((const __m128i*)(blk + 1)), 2), z);      /* 0, c1 .. c7 */
		__m128i b = _mm_cmpeq_epi16(_mm_loadu_si128((const __m128i*)(blk + 8)), z);
		unsigned k = ~(unsigned)_mm_movemask_epi8(_mm_packs_epi16(a, b));
		m |= zz_mask_tab[0][k & 254] | zz_mask_tab[1][k >> 8 & 255];
	}
	for (r = 2; r < 8; r += 2) {
		__m128i a = _mm_cmpeq_epi16(_mm_loadu_si128((const __m128i*)(blk + r * 8)), z);
		__m128i b = _mm_cmpeq_epi16(_mm_loadu_si128((const __m128i*)(blk + r * 8 + 8)), z);
		unsigned k = ~(unsigned)_mm_movemask_epi8(_mm_packs_epi16(a, b));
		m |= zz_mask_tab[r][k & 255] | zz_mask_tab[r + 1][k >> 8 & 255];
	}
#else
	for (r = 0; r < 8; r++) {
		unsigned k = 0; int c;
		for (c = r ? 0 : 1; c < 8; c++) k |= (unsigned)(blk[r * 8 + c] != 0) << c;
		m |= zz_mask_tab[r][k];
	}
#endif
	return m;
}

/* ---------------------------------------------------------------- in-memory "virtual" arrays */
struct jvirt_barray_control {
	JDIMENSION w, h;
	JBLOCKROW *rows;
	JBLOCK *data;
	struct jvirt_barray_control *next;
};

typedef struct {
	struct jpeg_memory_mgr pub;          /* must be first: cinfo.mem points here */
	struct jvirt_barray_control *head;
} jq_mem;

typedef struct {
	jq_mem mem;
	jpeg_component_info comps[MAX_COMPONENTS];
	JQUANT_TBL qt[NUM_QUANT_TBLS];
} jq_priv;

static jvirt_barray_ptr jq_request(j_common_ptr cinfo, int pool, boolean pre_zero, JDIMENSION w, JDIMENSION h,
		JDIMENSION maxaccess) {
	jq_mem *m = (jq_mem*)cinfo->mem; JDIMENSION y;
	struct jvirt_barray_control *a = (struct jvirt_barray_control*)calloc(1, sizeof(*a));
	(void)pool; (void)pre_zero; (void)maxaccess;
	if (!a) return NULL;
	a->w = w; a->h = h;
	a->rows = (JBLOCKROW*)malloc(sizeof(JBLOCKROW) * (h ? h : 1));
	a->data = (JBLOCK*)calloc((size_t)w * h + 1, sizeof(JBLOCK));
	if (!a->rows || !a->data) { free(a->rows); free(a->data); free(a); return NULL; }
	for (y = 0; y < h; y++) a->rows[y] = a->data + (size_t)y * w;
	a->next = m->head; m->head = a;
	return a;
}
static void jq_realize(j_common_ptr cinfo) { (void)cinfo; }
static JBLOCKARRAY jq_access(j_common_ptr cinfo, jvirt_barray_ptr a, JDIMENSION start, JDIMENSION n, boolean wr) {
	(void)cinfo; (void)n; (void)wr;
	return a->rows + start;
}

void jq_free(jq_image *im) {
	jq_priv *p = (jq_priv*)im->priv;
	while (im->markers) { jq_marker *m = im->markers; im->markers = m->next; free(m->data); free(m); }
	if (p) {
		while (p->mem.head) {
			struct jvirt_barray_control *a = p->mem.head; p->mem.head = a->next;
			free(a->rows); free(a->data); free(a);
		}
		free(p);
	}
	memset(im, 0, sizeof(*im));
}

/* ---------------------------------------------------------------- Huffman decoding */
typedef struct {
	int present;
	unsigned char bits[17], val[256];
	uint16_t look[512];                  /* 9-bit prefix -> (length << 8) | symbol, 0 = longer */
	int32_t maxcode[18], valptr[17], mincode[17];
	/* AC symbols whose code AND value bits fit in FAST_BITS: prefix -> (coefficient << 16) | (run << 4)
	 * | total bits, 0 = take the two-step path (long codes, EOB, ZRL).  One table read per symbol
	 * instead of code look-up -> value bits -> sign extension. */
	int32_t fast[1 << 10];
} jq_dhuff;
#define FAST_BITS 10

static int dhuff_build(jq_dhuff *h) {
	int code = 0, k = 0, l, i;
	memset(h->look, 0, sizeof(h->look));
	for (l = 1; l <= 16; l++) {
		h->valptr[l] = k; h->mincode[l] = code;
		for (i = 0; i < h->bits[l]; i++, k++, code++) {
			if (k >= 256) return -1;
			if (l <= 9) {
				int base = code << (9 - l), n = 1 << (9 - l), j;
				if (base + n > 512) return -1;
				for (j = 0; j < n; j++) h->look[base + j] = (uint16_t)((l << 8) | h->val[k]);
			}
		}
		h->maxcode[l] = h->bits[l] ? code - 1 : -1;
		if (code > (1 << l)) return -1;
		code <<= 1;
	}
	h->maxcode[17] = 0x7fffffff;
	for (i = 0; i < (1 << FAST_BITS); i++) {
		unsigned e = h->look[i >> (FAST_BITS - 9)]; int len = (int)(e >> 8), r = (int)(e >> 4) & 15, sz = (int)e & 15;
		h->fast[i] = 0;
		if (e && sz && len + sz <= FAST_BITS) {
			int v = (i >> (FAST_BITS - len - sz)) & ((1 << sz) - 1);
			if (v < (1 << (sz - 1))) v += 1 - (1 << sz);             /* F.2.2.1 EXTEND */
			h->fast[i] = (int32_t)((uint32_t)v << 16 | (uint32_t)r << 4 | (uint32_t)(len + sz));
		}
	}
	h->present = 1;
	return 0;
}

typedef struct {
	const unsigned char *p, *end;
	uint64_t buf; int nbits;
	int hit_marker;                      /* a marker (not a stuffed FF00) stopped the feed */
	int warn;                            /* bad Huffman codes met (decoding goes on, like libjpeg) */
	uint64_t fed;                        /* data bytes fed so far (an FF00 pair is one): 8 * fed - nbits = bit position */
} jq_bits;

static void bits_fill(jq_bits *b) {
	/* fast path: eight bytes ahead without an FF (no stuffing, no marker) are taken at once */
	if (!b->hit_marker && b->nbits <= 48 && b->end - b->p >= 8) {
		uint64_t x, nx; int k = (64 - b->nbits) >> 3;
		memcpy(&x, b->p, 8);
		nx = ~x;
		if (!((nx - 0x0101010101010101ULL) & ~nx & 0x8080808080808080ULL)) {
			uint64_t be = __builtin_bswap64(x);          /* little-endian hosts only (x86-64, aarch64) */
			b->buf = k == 8 ? be : (b->buf << (8 * k)) | (be >> (64 - 8 * k));
			b->p += k; b->nbits += 8 * k; b->fed += (unsigned)k;
			return;
		}
	}
	while (b->nbits <= 48) {
		unsigned c = 0;
		b->fed++;
		if (!b->hit_marker && b->p < b->end) {
			c = *b->p;
			if (c == 0xFF) {
				/* any number of FF fill bytes may precede a marker (B.1.1.2); like libjpeg's
				 * jpeg_fill_bit_buffer, FF..FF 00 reads as one stuffed FF.  A marker leaves p on the
				 * FF right before its code, where the restart and end-of-scan logic look for it. */
				const unsigned char *q = b->p + 1;
				while (q < b->end && *q == 0xFF) q++;
				if (q < b->end && *q == 0) b->p = q + 1;
				else { b->p = q - 1; b->hit_marker = 1; c = 0; }
			} else b->p++;
		}
		b->buf = (b->buf << 8) | c; b->nbits += 8;
	}
}
static inline unsigned bits_peek(jq_bits *b, int n) {
	if (b->nbits < n) bits_fill(b);
	return (unsigned)(b->buf >> (b->nbits - n)) & ((1u << n) - 1);
}
static inline unsigned bits_get(jq_bits *b, int n) {
	unsigned v;
	if (!n) return 0;
	v = bits_peek(b, n); b->nbits -= n;
	return v;
}
static inline int huff_decode(jq_bits *b, const jq_dhuff *h) {
	unsigned look = bits_peek(b, 16), e = h->look[look >> 7];
	int l, code;
	if (e) { b->nbits -= e >> 8; return e & 255; }
	for (l = 10; l <= 16; l++) {
		code = (int)(look >> (16 - l));
		if (code <= h->maxcode[l]) { b->nbits -= l; return h->val[h->valptr[l] + code - h->mincode[l]]; }
	}
	b->nbits -= 16; b->warn++;
	return 0;                            /* corrupt data: keep going like libjpeg's JWRN_HUFF_BAD_CODE path */
}
/* F.2.2.1 EXTEND without a branch (the sign of a coefficient is a coin toss): v < 2^(s-1) means negative */
static inline int extend(unsigned v, int s) {
	int neg = ((int)v - (1 << s >> 1)) >> 31;                /* all ones if v is in the lower half (and for s = 0) */
	return (int)v + (neg & (1 - (1 << s)));
}

/* ---------------------------------------------------------------- the reader */
static int codec_thread_count(void);
typedef struct {
	int ncomp, ci[4], td[4], ta[4], Ss, Se, Ah, Al;
} jq_scan;

typedef struct {
	jq_image *im; jq_priv *pv;
	jq_dhuff dc[4], ac[4];
	int pred[MAX_COMPONENTS];
	unsigned eobrun;
	JDIMENSION mcux, mcuy;
	int ri;                              /* restart interval in force for the scan being decoded */
	int warn;                            /* recoverable anomalies met while decoding (added to jq_image.warnings by jq_read) */
} jq_dec;

static void dec_block_seq(jq_dec *d, jq_bits *b, const jq_scan *s, int k, JCOEFPTR blk) {
	int c = s->ci[k], t, i;
	const jq_dhuff *h = &d->ac[s->ta[k]];
	uint64_t buf; int nbits;
	t = huff_decode(b, &d->dc[s->td[k]]);
	d->pred[c] += extend(bits_get(b, t & 15), t & 15);
	blk[0] = (JCOEF)d->pred[c];
	buf = b->buf; nbits = b->nbits;                     /* the bit window lives in registers inside the loop */
	for (i = 1; i < 64; ) {
		/* one refill check per symbol: a code (<= 16 bits) and its value bits (<= 15) fit in 32 */
		unsigned look, e, v; int rs, r, sz, f;
		if (nbits < 32) { b->buf = buf; b->nbits = nbits; bits_fill(b); buf = b->buf; nbits = b->nbits; }
		look = (unsigned)(buf >> (nbits - 16)) & 0xFFFF;
		f = h->fast[look >> (16 - FAST_BITS)];
		if (f) {                                        /* code and value in one step */
			i += (f >> 4) & 15; nbits -= f & 15;
			blk[zz_nat[i]] = (JCOEF)(f >> 16);
			i++;
			continue;
		}
		e = h->look[look >> 7];
		if (e) { nbits -= (int)(e >> 8); rs = (int)(e & 255); }
		else { b->buf = buf; b->nbits = nbits; rs = huff_decode(b, h); nbits = b->nbits; }
		r = rs >> 4; sz = rs & 15;
		if (!sz) { if (r != 15) break; i += 16; continue; }
		i += r;
		v = (unsigned)(buf >> (nbits - sz)) & ((1u << sz) - 1); nbits -= sz;
		blk[zz_nat[i]] = (JCOEF)extend(v, sz);
		i++;
	}
	b->buf = buf; b->nbits = nbits;
}

static void dec_block_prog(jq_dec *d, jq_bits *b, const jq_scan *s, int k, JCOEFPTR blk) {
	int c = s->ci[k], Al = s->Al, i;
	if (s->Ss == 0) {                                   /* DC scans, G.1.2.1 */
		if (s->Ah == 0) {
			int t = huff_decode(b, &d->dc[s->td[k]]);
			d->pred[c] += extend(bits_get(b, t & 15), t & 15);
			blk[0] = (JCOEF)(d->pred[c] * (1 << Al));
		} else if (bits_get(b, 1)) blk[0] |= (JCOEF)(1 << Al);
		return;
	}
	if (s->Ah == 0) {                                   /* AC first scan, G.1.2.2 */
		if (d->eobrun) { d->eobrun--; return; }
		for (i = s->Ss; i <= s->Se; ) {
			int rs = huff_decode(b, &d->ac[s->ta[k]]), r = rs >> 4, sz = rs & 15;
			if (sz) {
				i += r;
				blk[zz_nat[i]] = (JCOEF)(extend(bits_get(b, sz), sz) * (1 << Al));
				i++;
			} else if (r == 15) i += 16;
			else { d->eobrun = (1u << r) + bits_get(b, r) - 1; break; }
		}
		return;
	}
	{                                                   /* AC refinement scan, G.1.2.3 */
		/* The coefficients that are already non-zero (they take a correction bit each) come from a
		 * bit mask of the block instead of a walk over up to 63 positions: in these scans most
		 * blocks are visited only to pass an end-of-band run or a handful of coefficients. */
		int p1 = 1 << Al, m1 = -(1 << Al), Se = s->Se;
		const uint64_t range = (Se == 63 ? ~0ULL : (1ULL << (Se + 1)) - 1) & (~0ULL << s->Ss);
		const uint64_t nz = nonzero_mask_zz_ac(blk) & range;
		uint64_t w;
#define REFINE(w_) while (w_) { JCOEFPTR cp = blk + zz_nat[__builtin_ctzll(w_)]; w_ &= w_ - 1; \
		if (bits_get(b, 1) && !(*cp & p1)) *cp += (JCOEF)(*cp >= 0 ? p1 : m1); }
		i = s->Ss;
		if (!d->eobrun) {
			while (i <= Se) {
				int rs = huff_decode(b, &d->ac[s->ta[k]]), r = rs >> 4, sz = rs & 15, val = 0, t;
				uint64_t zeros;
				if (sz) val = bits_get(b, 1) ? p1 : m1;
				else if (r != 15) { d->eobrun = (1u << r) + bits_get(b, r); break; }
				/* skip r zero-history coefficients; the non-zero ones on the way take a correction bit */
				zeros = ~nz & range & (~0ULL << i);
				for (; r > 0 && zeros; r--) zeros &= zeros - 1;
				t = zeros ? __builtin_ctzll(zeros) : Se + 1;             /* where the new coefficient goes */
				w = nz & (~0ULL << i) & (t > 63 ? ~0ULL : (1ULL << t) - 1);
				REFINE(w)
				i = t;
				if (val && i <= Se) blk[zz_nat[i]] = (JCOEF)val;
				i++;
			}
		}
		if (d->eobrun) {
			if (i <= Se) { w = nz & (~0ULL << i); REFINE(w) }
			d->eobrun--;
		}
#undef REFINE
	}
}

/* ---------------------------------------------------------------- sequential scans on several threads
 * An entropy-coded segment has no entry points, but Huffman-coded JPEG data re-synchronizes: a
 * decoder started at an arbitrary byte soon reads the same codes at the same bit positions as the
 * true one.  A sequential (SOF0/SOF1) scan without restart markers is therefore decoded in
 * three steps:
 *   1. the segment is cut into chunks; each thread PARSES its chunk from the first byte as if an
 *      MCU started there (codes only, no coefficients stored) and notes the bit position of
 *      every MCU it believes to start;
 *   2. one thread walks the chunks in order: from the true end of chunk k it parses on until
 *      its MCU start coincides with one noted by the thread of a later chunk - same bit
 *      position, same decoder state (start of an MCU; DC predictors do not influence parsing),
 *      so from there on that thread's notes are the truth, and the MCU number of that point is
 *      known;
 *   3. each thread decodes for real, from one synchronization point to the next, into the
 *      coefficient arrays: the MCU numbers are known now, and so are the DC predictors (steps 1
 *      and 2 add up the DC differences they pass; the sums are checked against what step 3
 *      arrives at).
 * With restart markers (DRI) the intervals are independent by definition: step 3 alone, one
 * range per interval, nothing to guess.
 * Anything unexpected (a marker inside the data, positions that do not line up, too few bits,
 * restart markers missing or out of sequence) abandons the attempt: the arrays of the scan are
 * cleared and the plain decoder runs, so damaged files behave as before.  A chunk that never
 * synchronizes is simply decoded by its predecessor.  Results are identical to the one-thread
 * decoder by construction (step 3 runs the same block decoder on the same bits); tests/test_cli.py
 * compares the files on every flavour and thread count. */
#define PAR_MIN_BYTES (128 << 10)        /* shorter segments are not worth the threads (JPEGQS_PAR_MIN_BYTES: test knob) */
#define PAR_MIN_THREADS 4                /* steps 1 + 3 read the data twice: two threads would be slower than one */
#define PAR_MAX_CHUNKS 64

typedef struct { const jq_dhuff *dc, *ac; int k, h, v, hs, vs; } jq_mcu_blk;    /* scan component k, block (h, v) of the MCU */

typedef struct {
	const unsigned char *p, *end;        /* raw bytes of the range */
	int skip_bits;                       /* bits of the first byte that belong to the MCU before */
	uint64_t fed0;                       /* data-byte index of p (bit positions are 8 * fed - nbits) */
	uint64_t m0, m1;                     /* MCUs [m0, m1) */
	uint64_t end_pos;                    /* bit position the range must end at (0: not checked) */
	int pred0[4];                        /* DC predictors of the scan's components at m0 */
	int endpred[4], check_pred, warn;    /* ... and at m1 (must be the next range's pred0 if check_pred) */
} jq_range;

typedef struct {
	jq_dec *d; const jq_scan *s;
	const unsigned char *seg, *segend;               /* entropy-coded bytes, up to the next marker */
	jq_mcu_blk blk[MAX_COMPONENTS * 16]; int nblk;   /* the blocks of one MCU */
	JDIMENSION nx; uint64_t nmcu;
	int nchunk;
	const unsigned char *cstart[PAR_MAX_CHUNKS + 1]; /* raw chunk starts (cstart[nchunk] = segend) */
	uint64_t cbase[PAR_MAX_CHUNKS + 1];              /* data-byte index of each chunk start */
	uint64_t *pos[PAR_MAX_CHUNKS]; size_t npos[PAR_MAX_CHUNKS];   /* step 1: MCU start bit positions ... */
	int32_t *dcs[PAR_MAX_CHUNKS];                    /* ... and the sums of the DC differences up to each (4 per entry) */
	jq_range *range; int nrange;
	int phase;                                       /* what the workers do: 1 parse, 3 decode */
	uint64_t stitched;                               /* MCUs the stitching thread had to parse itself */
	volatile int next, fail;
} jq_par;

static inline uint64_t par_pos(const jq_bits *b) { return 8 * b->fed - (unsigned)b->nbits; }

/* parses one block without storing anything (same table walk as dec_block_seq) */
static inline int skip_block(jq_bits *b, const jq_dhuff *dc, const jq_dhuff *h) {
	uint64_t buf; int nbits, i, t, diff;
	t = huff_decode(b, dc);
	diff = extend(bits_get(b, t & 15), t & 15);
	buf = b->buf; nbits = b->nbits;
	for (i = 1; i < 64; ) {
		unsigned look, e; int rs, r, sz, f;
		if (nbits < 32) { b->buf = buf; b->nbits = nbits; bits_fill(b); buf = b->buf; nbits = b->nbits; }
		look = (unsigned)(buf >> (nbits - 16)) & 0xFFFF;
		f = h->fast[look >> (16 - FAST_BITS)];
		if (f) { i += ((f >> 4) & 15) + 1; nbits -= f & 15; continue; }
		e = h->look[look >> 7];
		if (e) { nbits -= (int)(e >> 8); rs = (int)(e & 255); }
		else { b->buf = buf; b->nbits = nbits; rs = huff_decode(b, h); nbits = b->nbits; }
		r = rs >> 4; sz = rs & 15;
		if (!sz) { if (r != 15) break; i += 16; continue; }
		i += r + 1; nbits -= sz;
	}
	b->buf = buf; b->nbits = nbits;
	return diff;
}
/* parses one MCU; dc[k] += the DC differences of the scan's component k */
static inline void skip_mcu(const jq_par *q, jq_bits *b, int32_t *dc) {
	int k;
	for (k = 0; k < q->nblk; k++) dc[q->blk[k].k] += skip_block(b, q->blk[k].dc, q->blk[k].ac);
}

/* a reader at bit position pos, reached from the start of chunk c (which must not lie behind it) */
static int par_reader_at(const jq_par *q, int c, uint64_t pos, jq_bits *b, const unsigned char **raw) {
	const unsigned char *p = q->cstart[c]; uint64_t idx = q->cbase[c], want = pos >> 3;
	if (want < idx) return -1;
	while (idx < want) {                                /* an FF00 pair is one data byte */
		if (p >= q->segend) return -1;
		p += p[0] == 0xFF ? 2 : 1; idx++;
	}
	if (raw) *raw = p;
	if (b) {
		memset(b, 0, sizeof(*b));
		b->p = p; b->end = q->segend; b->fed = idx;
		if (pos & 7) bits_get(b, (int)(pos & 7));
	}
	return 0;
}

/* step 1 */
static void par_parse_chunk(jq_par *q, int c) {
	jq_bits b; size_t cap = 4096, n = 0; uint64_t *v = (uint64_t*)malloc(cap * sizeof(*v)), limit = 8 * q->cbase[c + 1];
	int32_t *s = (int32_t*)malloc(cap * 4 * sizeof(*s)), cum[4] = { 0, 0, 0, 0 };
	memset(&b, 0, sizeof(b)); b.p = q->cstart[c]; b.end = q->segend; b.fed = q->cbase[c];
	while (v && s) {
		uint64_t pos = par_pos(&b);
		if (n == cap) {
			uint64_t *w = (uint64_t*)realloc(v, 2 * cap * sizeof(*v)); int32_t *t;
			if (!w) { free(v); v = NULL; break; }
			v = w;
			t = (int32_t*)realloc(s, 2 * cap * 4 * sizeof(*s));
			if (!t) { free(s); s = NULL; break; }
			s = t; cap *= 2;
		}
		memcpy(s + 4 * n, cum, sizeof(cum));
		v[n++] = pos;                                   /* the last entry: first MCU start at or beyond the chunk end */
		if (pos >= limit) break;
		/* a chunk with 16 times its share of the image's MCUs is crafted or nonsense: bound the notes */
		if (n > 16 * (q->nmcu / (unsigned)q->nchunk) + 4096) { free(v); v = NULL; break; }
		skip_mcu(q, &b, cum);
	}
	if (!v || !s) { free(v); free(s); v = NULL; s = NULL; q->fail = 1; n = 0; }
	q->pos[c] = v; q->dcs[c] = s; q->npos[c] = n;
}

/* step 2: fills q->range; returns 0, or -1 if the data does not hold nmcu MCUs */
static int par_stitch(jq_par *q) {
	uint64_t endbits = 8 * q->cbase[q->nchunk], m = 0;
	int cur = 0, k; size_t idx = 0; jq_range *r; int32_t pred[4] = { 0, 0, 0, 0 };      /* DC predictors at MCU m */
	q->nrange = 0;
	r = &q->range[q->nrange++];
	memset(r, 0, sizeof(*r)); r->p = q->seg; r->end = q->segend; r->m0 = 0;
	for (;;) {
		/* the notes of chunk `cur` are true from entry idx (= MCU m) to the last one */
		uint64_t E, mE; jq_bits b; int j; size_t pj, last;
		if (!q->npos[cur]) return -1;
		last = q->npos[cur] - 1;
		E = q->pos[cur][last]; mE = m + (uint64_t)(last - idx);
		if (mE >= q->nmcu) break;                       /* the image ends inside this chunk */
		for (k = 0; k < 4; k++) pred[k] += q->dcs[cur][4 * last + k] - q->dcs[cur][4 * idx + k];
		if (E > endbits) return -1;
		for (j = cur + 1; j < q->nchunk && E >= 8 * q->cbase[j + 1]; j++);
		if (j >= q->nchunk) return -1;                  /* MCUs are missing and no data is left */
		if (par_reader_at(q, j, E, &b, NULL)) return -1;
		m = mE; pj = 0;
		for (;;) {
			uint64_t P = par_pos(&b);
			if (P > endbits) return -1;
			while (j + 1 < q->nchunk && P >= 8 * q->cbase[j + 1]) { j++; pj = 0; }
			while (pj < q->npos[j] && q->pos[j][pj] < P) pj++;
			if (pj < q->npos[j] && q->pos[j][pj] == P) break;           /* synchronized with chunk j */
			if (m >= q->nmcu) break;
			if (q->stitched > q->nmcu / 8 + 256) return -1;             /* the chunks do not synchronize: not worth it */
			skip_mcu(q, &b, pred); m++; q->stitched++;
		}
		if (m >= q->nmcu) break;                        /* this one thread parsed to the end of the image */
		{                                               /* a new range starts at chunk j's entry pj = MCU m */
			uint64_t P = q->pos[j][pj]; const unsigned char *raw;
			if (par_reader_at(q, j, P, NULL, &raw)) return -1;
			r->m1 = m; r->end_pos = P; r->check_pred = 1;
			r = &q->range[q->nrange++];
			memset(r, 0, sizeof(*r));
			r->p = raw; r->end = q->segend; r->skip_bits = (int)(P & 7); r->fed0 = P >> 3; r->m0 = m;
			for (k = 0; k < 4; k++) r->pred0[k] = pred[k];
			cur = j; idx = pj;
		}
	}
	r->m1 = q->nmcu;
	return 0;
}

static inline JCOEFPTR par_block(const jq_par *q, const jq_mcu_blk *mb, JDIMENSION x, JDIMENSION y) {
	return q->d->im->coef_arrays[q->s->ci[mb->k]]->rows[y * (JDIMENSION)mb->vs + (JDIMENSION)mb->v][x * (JDIMENSION)mb->hs + (JDIMENSION)mb->h];
}

/* step 3 */
/* ld: the worker's private copy of the decoder state (tables + predictors) */
static void par_decode_range(jq_par *q, jq_range *r, jq_dec *ld) {
	jq_bits b; uint64_t m; int k;
	memset(ld->pred, 0, sizeof(ld->pred));
	for (k = 0; k < q->s->ncomp; k++) ld->pred[q->s->ci[k]] = r->pred0[k];
	memset(&b, 0, sizeof(b)); b.p = r->p; b.end = r->end; b.fed = r->fed0;
	if (r->skip_bits) bits_get(&b, r->skip_bits);
	for (m = r->m0; m < r->m1; m++) {
		JDIMENSION y = (JDIMENSION)(m / q->nx), x = (JDIMENSION)(m % q->nx);
		for (k = 0; k < q->nblk; k++) dec_block_seq(ld, &b, q->s, q->blk[k].k, par_block(q, &q->blk[k], x, y));
	}
	if (r->end_pos && par_pos(&b) != r->end_pos) q->fail = 1;
	for (k = 0; k < q->s->ncomp; k++) r->endpred[k] = ld->pred[q->s->ci[k]];
	r->warn = b.warn;
}

static void *par_worker(void *arg) {
	jq_par *q = (jq_par*)arg; jq_dec *ld = NULL;
	if (q->phase == 3) {
		ld = (jq_dec*)malloc(sizeof(*ld));
		if (!ld) { q->fail = 1; return NULL; }
		memcpy(ld, q->d, sizeof(*ld));
	}
	for (;;) {
		int i = __sync_fetch_and_add(&q->next, 1);
		if (q->phase == 1) { if (i >= q->nchunk) break; par_parse_chunk(q, i); }
		else { if (i >= q->nrange) break; par_decode_range(q, &q->range[i], ld); }
	}
	free(ld);
	return NULL;
}
static void par_run(jq_par *q, int phase, int nthr) {
	pthread_t tid[64]; int i, started = 0;
	q->phase = phase; q->next = 0;
	for (i = 1; i < nthr && i < 64; i++) { if (pthread_create(&tid[started], NULL, par_worker, q)) break; started++; }
	par_worker(q);
	for (i = 0; i < started; i++) pthread_join(tid[i], NULL);
}

/* 1 = the scan was decoded here (*next set), 0 = not applicable / abandoned (arrays of the scan cleared
 * again): the caller runs the plain decoder */
static int dec_scan_parallel(jq_dec *d, const jq_scan *s, const unsigned char *p, const unsigned char *end,
		const unsigned char **next) {
	jq_image *im = d->im; jq_par *q; int nthr = codec_thread_count(), k, h, v, ri = d->ri, ok = 0, i;
	const unsigned char *t, *segend = NULL; uint64_t stuffed = 0; size_t len, min_bytes = PAR_MIN_BYTES, chunk_min;
	const char *env = getenv("JPEGQS_PAR_MIN_BYTES"); double tm[4] = { 0 };
	JDIMENSION ny;
	if (env && atoi(env) > 0) min_bytes = (size_t)atoi(env);
	chunk_min = min_bytes / 4 < 64 ? 64 : min_bytes / 4;
	if (im->progressive || nthr < PAR_MIN_THREADS || (size_t)(end - p) < min_bytes || getenv("JPEGQS_SERIAL_DECODE")) return 0;
	q = (jq_par*)calloc(1, sizeof(*q));
	if (!q) return 0;
	q->d = d; q->s = s; q->seg = p;
	/* the blocks of an MCU (A.2.3; a one-component scan is not interleaved: MCU = one block) */
	if (s->ncomp == 1) {
		jpeg_component_info *c = &im->cinfo.comp_info[s->ci[0]];
		q->nx = c->width_in_blocks; ny = c->height_in_blocks;
		q->blk[0].dc = &d->dc[s->td[0]]; q->blk[0].ac = &d->ac[s->ta[0]]; q->blk[0].hs = q->blk[0].vs = 1;
		q->nblk = 1;
	} else {
		q->nx = d->mcux; ny = d->mcuy;
		for (k = 0; k < s->ncomp; k++) {
			jpeg_component_info *c = &im->cinfo.comp_info[s->ci[k]];
			for (v = 0; v < c->v_samp_factor; v++) for (h = 0; h < c->h_samp_factor; h++) {
				jq_mcu_blk *mb;
				if (q->nblk >= (int)(sizeof(q->blk) / sizeof(q->blk[0]))) goto out;
				mb = &q->blk[q->nblk++];
				mb->dc = &d->dc[s->td[k]]; mb->ac = &d->ac[s->ta[k]]; mb->k = k; mb->h = h; mb->v = v;
				mb->hs = c->h_samp_factor; mb->vs = c->v_samp_factor;
			}
		}
	}
	q->nmcu = (uint64_t)q->nx * ny;
	if (!q->nmcu) goto out;
	if (!ri) {
		/* A parser that starts inside an MCU finds its place because the blocks of an MCU do not all
		 * use the same Huffman tables: with the wrong block phase it soon reads nonsense and falls
		 * back into step at an MCU start.  If the table sequence of the MCU repeats with a shorter
		 * period (CMYK or RGB files with one table pair, say) it would stay in step with the bits
		 * and out of phase with the MCUs for good: those scans are left to the one-thread decoder. */
		int per;
		for (per = 1; per < q->nblk; per++) {
			if (q->nblk % per) continue;
			for (k = per; k < q->nblk; k++) {
				const jq_dhuff *a = q->blk[k].dc, *b = q->blk[k - per].dc, *c = q->blk[k].ac, *e = q->blk[k - per].ac;
				if (memcmp(a->bits, b->bits, 17) || memcmp(a->val, b->val, 256) || memcmp(c->bits, e->bits, 17) || memcmp(c->val, e->val, 256)) break;
			}
			if (k == q->nblk) goto out;
		}
	}

	if (ri) {
		/* restart intervals: ceil(nmcu / ri) - 1 markers RST0, RST1, ... RST7, RST0 ... and nothing else */
		uint64_t nint = (q->nmcu + (unsigned)ri - 1) / (unsigned)ri, j = 0;
		if (nint > (1u << 24)) goto out;
		q->range = (jq_range*)calloc((size_t)nint, sizeof(jq_range));
		if (!q->range) goto out;
		q->range[0].p = p;
		for (t = p; (t = (const unsigned char*)memchr(t, 0xFF, (size_t)(end - t))) != NULL; ) {
			const unsigned char *u = t + 1;
			while (u < end && *u == 0xFF) u++;          /* fill bytes before a marker: the range ends at the first */
			if (u >= end) { segend = t; break; }
			if (*u == 0) { if (u > t + 1) goto out; t += 2; continue; }    /* FF..FF 00: left to the plain decoder */
			if ((*u & 0xF8) == 0xD0) {
				if (j + 1 >= nint || (unsigned)(*u & 7) != (unsigned)(j & 7)) goto out;
				q->range[j].end = t; j++; q->range[j].p = u + 1;
				t = u + 1; continue;
			}
			segend = t; break;
		}
		if (!segend || j + 1 != nint) goto out;
		q->range[j].end = segend;
		for (j = 0; j < nint; j++) {
			q->range[j].m0 = j * (unsigned)ri;
			q->range[j].m1 = (j + 1) * (unsigned)ri < q->nmcu ? (j + 1) * (unsigned)ri : q->nmcu;
		}
		q->nrange = (int)nint; q->segend = segend;
		par_run(q, 3, nthr);
		if (q->fail) goto clear;
		for (i = 0; i < q->nrange; i++) d->warn += q->range[i].warn;
		if (getenv("JPEGQS_CODEC_TRACE"))
			fprintf(stderr, "jpegcoef: scan decoded on %d threads: %d restart intervals\n", nthr, q->nrange);
		*next = segend; ok = 1;
		goto out;
	}

	/* the segment ends at the first FF that is not followed by 00; it and any fill bytes after it must
	 * lead to a real marker */
	for (t = p; (t = (const unsigned char*)memchr(t, 0xFF, (size_t)(end - t))) != NULL; ) {
		if (t + 1 < end && t[1] == 0) { t += 2; continue; }
		segend = t; break;
	}
	if (!segend) goto out;
	for (t = segend + 1; t < end && *t == 0xFF; t++);
	if (t >= end || *t == 0 || (*t & 0xF8) == 0xD0) goto out;
	len = (size_t)(segend - p);
	if (len < min_bytes) goto out;
	q->segend = segend;
	q->nchunk = nthr * 2 < PAR_MAX_CHUNKS ? nthr * 2 : PAR_MAX_CHUNKS;
	if ((size_t)q->nchunk > len / chunk_min) q->nchunk = (int)(len / chunk_min);
	if (q->nchunk < 2) goto out;
	/* chunk starts: never between the FF and the 00 of a stuffed byte; data-byte index of each */
	t = p;
	for (i = 0; i < q->nchunk; i++) {
		const unsigned char *c = p + (size_t)((uint64_t)len * (unsigned)i / (unsigned)q->nchunk);
		if (c < t) c = t;
		while (c > p && c < segend && c[-1] == 0xFF) c++;
		for (; t < c; ) {                               /* stuffed bytes before c */
			const unsigned char *f = (const unsigned char*)memchr(t, 0xFF, (size_t)(c - t));
			if (!f) break;
			stuffed++; t = f + 2;                       /* inside the segment every FF is followed by 00 */
		}
		if (t < c) t = c;
		q->cstart[i] = c; q->cbase[i] = (uint64_t)(c - p) - stuffed;
	}
	for (; t < segend; ) {
		const unsigned char *f = (const unsigned char*)memchr(t, 0xFF, (size_t)(segend - t));
		if (!f) break;
		stuffed++; t = f + 2;
	}
	q->cstart[q->nchunk] = segend; q->cbase[q->nchunk] = (uint64_t)len - stuffed;
	for (i = 0; i < q->nchunk; i++) if (q->cbase[i + 1] <= q->cbase[i]) goto out;

	q->range = (jq_range*)calloc((size_t)q->nchunk + 1, sizeof(jq_range));
	if (!q->range) goto out;
	tm[0] = trace_ms();
	par_run(q, 1, nthr);
	tm[1] = trace_ms();
	if (q->fail || par_stitch(q)) goto out;             /* nothing was written to the arrays yet */
	tm[2] = trace_ms();
	par_run(q, 3, nthr);
	tm[3] = trace_ms();
	if (q->fail) goto clear;
	for (i = 0; i < q->nrange; i++) {                   /* the predictors step 2 worked out must be the ones step 3 arrived at */
		if (i + 1 < q->nrange && q->range[i].check_pred)
			for (k = 0; k < s->ncomp; k++) if (q->range[i].endpred[k] != q->range[i + 1].pred0[k]) goto clear;
		d->warn += q->range[i].warn;
	}
	if (getenv("JPEGQS_CODEC_TRACE"))
		fprintf(stderr, "jpegcoef: scan decoded on %d threads: %d chunks, %d ranges, %llu of %llu MCUs parsed while stitching; "
				"parse %.1f ms, stitch %.1f ms, decode %.1f ms\n",
				nthr, q->nchunk, q->nrange, (unsigned long long)q->stitched, (unsigned long long)q->nmcu,
				tm[1] - tm[0], tm[2] - tm[1], tm[3] - tm[2]);
	*next = segend; ok = 1;
	goto out;
clear:
	if (getenv("JPEGQS_CODEC_TRACE")) fprintf(stderr, "jpegcoef: threaded decode abandoned, decoding again on one thread\n");
	for (k = 0; k < s->ncomp; k++) {
		jvirt_barray_ptr a = im->coef_arrays[s->ci[k]];
		memset(a->data, 0, (size_t)a->w * a->h * sizeof(JBLOCK));
	}
out:
	for (i = 0; i < PAR_MAX_CHUNKS; i++) { free(q->pos[i]); free(q->dcs[i]); }
	free(q->range); free(q);
	return ok;
}


static int dec_scan(jq_dec *d, const jq_scan *s, const unsigned char *p, const unsigned char *end,
		const unsigned char **next, char *err) {
	jq_image *im = d->im; jq_bits b; int prog = im->progressive, k, ri = d->ri;
	JDIMENSION nx, ny, x, y; unsigned count = 0, rst = 0;
	memset(&b, 0, sizeof(b)); b.p = p; b.end = end;
	memset(d->pred, 0, sizeof(d->pred)); d->eobrun = 0;
	for (k = 0; k < s->ncomp; k++) {
		int need_dc = !prog || (s->Ss == 0 && s->Ah == 0), need_ac = prog ? s->Ss > 0 : 1;
		if ((need_dc && !d->dc[s->td[k]].present) || (need_ac && !d->ac[s->ta[k]].present)) {
			snprintf(err, 256, "scan uses an undefined Huffman table"); return -1;
		}
	}
	if (dec_scan_parallel(d, s, p, end, next)) return 0;
	if (s->ncomp == 1) {
		jpeg_component_info *c = &im->cinfo.comp_info[s->ci[0]];
		nx = c->width_in_blocks; ny = c->height_in_blocks;
	} else { nx = d->mcux; ny = d->mcuy; }
	for (y = 0; y < ny; y++) for (x = 0; x < nx; x++) {
		if (ri && count == (unsigned)ri) {              /* restart: align, expect RSTn (B.2.1, F.2.2.5) */
			b.nbits = 0; b.buf = 0;
			if (!b.hit_marker) {                        /* skip padding up to the marker */
				while (b.p + 1 < b.end && !(b.p[0] == 0xFF && b.p[1] != 0 && b.p[1] != 0xFF)) b.p++;
			}
			if (b.p + 1 < b.end && b.p[0] == 0xFF && (b.p[1] & 0xF8) == 0xD0) b.p += 2;
			b.hit_marker = 0; rst++; count = 0;
			memset(d->pred, 0, sizeof(d->pred)); d->eobrun = 0;
		}
		count++;
		if (s->ncomp == 1) {
			JCOEFPTR blk = im->coef_arrays[s->ci[0]]->rows[y][x];
			if (prog) dec_block_prog(d, &b, s, 0, blk); else dec_block_seq(d, &b, s, 0, blk);
		} else for (k = 0; k < s->ncomp; k++) {
			jpeg_component_info *c = &im->cinfo.comp_info[s->ci[k]]; int h, v;
			for (v = 0; v < c->v_samp_factor; v++) for (h = 0; h < c->h_samp_factor; h++) {
				JCOEFPTR blk = im->coef_arrays[s->ci[k]]->rows[y * c->v_samp_factor + v][x * c->h_samp_factor + h];
				if (prog) dec_block_prog(d, &b, s, k, blk); else dec_block_seq(d, &b, s, k, blk);
			}
		}
	}
	/* position of the next marker */
	if (!b.hit_marker) {
		const unsigned char *q = b.p;
		while (q + 1 < end && !(q[0] == 0xFF && q[1] != 0 && q[1] != 0xFF && (q[1] & 0xF8) != 0xD0)) q++;
		*next = q;
	} else *next = b.p;
	(void)rst;
	d->warn += b.warn;
	return 0;
}


/* ---------------------------------------------------------------- progressive scans side by side
 * The scans of a progressive file are independent unless they touch the same coefficients: a
 * scan waits for the earlier scans of one of its components whose band [Ss, Se] overlaps its own
 * (the first scan of a band, then its refinements), and an AC refinement scan - which looks at
 * the whole AC part of a block to find the coefficients that are already non-zero - is ordered
 * against every other AC scan of its component.  jq_read first only RECORDS the scans (the
 * Huffman tables and restart interval in force, the bytes up to the next marker), then worker
 * threads decode them as they become ready.  If a scan does not end where the next marker was
 * found, or anything else goes wrong, the file is read again the plain way, scan after scan, so
 * damaged files keep their behaviour (and their messages). */
#define JQ_MAX_DEFER 64
typedef struct {
	jq_scan s; jq_dec *d;                /* d: a copy of the decoder state (tables) at the scan's SOS */
	const unsigned char *p, *segend;
	uint64_t deps;                       /* earlier scans that must be complete */
	int started, done, rc;
} jq_dscan;
typedef struct {
	jq_dscan *sc; int n; const unsigned char *end;
	pthread_mutex_t mu; pthread_cond_t cv;
	int bad;
} jq_sched;

static void *sched_worker(void *arg) {
	jq_sched *q = (jq_sched*)arg; int i; char err[256];
	pthread_mutex_lock(&q->mu);
	for (;;) {
		int pick = -1, unstarted = 0;
		for (i = 0; i < q->n; i++) {
			uint64_t dm = q->sc[i].deps; int k, ready = 1;
			if (q->sc[i].started) continue;
			unstarted = 1;
			for (k = 0; k < i && ready; k++) if ((dm >> k & 1) && !q->sc[k].done) ready = 0;
			if (ready) { pick = i; break; }
		}
		if (pick < 0) {
			if (!unstarted || q->bad) break;
			pthread_cond_wait(&q->cv, &q->mu);
			continue;
		}
		q->sc[pick].started = 1;
		pthread_mutex_unlock(&q->mu);
		{
			jq_dscan *c = &q->sc[pick]; const unsigned char *next = NULL;
			c->rc = dec_scan(c->d, &c->s, c->p, q->end, &next, err);
			if (c->rc || next != c->segend) c->rc = -1;
		}
		pthread_mutex_lock(&q->mu);
		q->sc[pick].done = 1;
		if (q->sc[pick].rc) q->bad = 1;
		pthread_cond_broadcast(&q->cv);
	}
	pthread_mutex_unlock(&q->mu);
	return NULL;
}

/* 0 = all scans decoded as recorded (warnings added up), -1 = read the file again the plain way */
static int sched_run(jq_image *im, jq_dscan *sc, int n, const unsigned char *end) {
	jq_sched q; pthread_t tid[64]; int i, j, k, nthr = codec_thread_count(), started = 0, rc = 0;
	memset(&q, 0, sizeof(q));
	q.sc = sc; q.n = n; q.end = end;
	for (j = 0; j < n; j++) for (i = 0; i < j; i++) {
		const jq_scan *a = &sc[i].s, *b = &sc[j].s; int share = 0;
		for (k = 0; k < a->ncomp; k++) { int m; for (m = 0; m < b->ncomp; m++) if (a->ci[k] == b->ci[m]) share = 1; }
		if (!share) continue;
		if ((a->Ss <= b->Se && b->Ss <= a->Se) ||
				(a->Ss > 0 && b->Ss > 0 && (a->Ah > 0 || b->Ah > 0))) sc[j].deps |= 1ULL << i;
	}
	pthread_mutex_init(&q.mu, NULL); pthread_cond_init(&q.cv, NULL);
	if (nthr > n) nthr = n;
	for (i = 1; i < nthr && i < 64; i++) { if (pthread_create(&tid[started], NULL, sched_worker, &q)) break; started++; }
	sched_worker(&q);
	for (i = 0; i < started; i++) pthread_join(tid[i], NULL);
	pthread_cond_destroy(&q.cv); pthread_mutex_destroy(&q.mu);
	for (i = 0; i < n; i++) { if (!sc[i].done || sc[i].rc) rc = -1; else im->warnings += sc[i].d->warn; }
	if (!rc && getenv("JPEGQS_CODEC_TRACE")) fprintf(stderr, "jpegcoef: %d progressive scans decoded on %d threads\n", n, started + 1);
	return rc;
}

static unsigned be16(const unsigned char *p) { return (unsigned)p[0] << 8 | p[1]; }

/* The first marker at or after p that is not RSTn (an FF followed by neither 00, FF nor D0..D7), or
 * end - 1 when none follows: the markers-only walk's skip over entropy-coded data.  memchr finds the
 * FF bytes, so the walk over an 8K file costs about a millisecond. */
static const unsigned char *next_marker(const unsigned char *p, const unsigned char *end) {
	while (p + 1 < end) {
		const unsigned char *q = (const unsigned char*)memchr(p, 0xFF, (size_t)(end - 1 - p));
		if (!q) return end - 1;
		if (q[1] != 0 && q[1] != 0xFF && (q[1] & 0xF8) != 0xD0) return q;
		p = q + 1;
	}
	return p;
}

/* defer: progressive scans are recorded and decoded side by side at the end (returns 1 if that did
 * not work out: the caller reads the file again with defer = 0) */
typedef struct { jq_scanrec *recs; int cap, n; } jq_recs;      /* jq_read_scans' record of the scans */

static int jq_read_impl(const unsigned char *data, size_t len, int copy, jq_image *im, char *err, int defer,
		jq_header *hdr, int skip_data, jq_recs *rec) {
	const unsigned char *p = data, *end = data + len;
	jq_priv *pv; jq_dec *d; jq_marker **tail; int have_frame = 0, i, done = 0, adobe = -1;
	jq_dscan *dsc = NULL; int ndsc = 0, retry = 0, sof_code = 0;
	memset(im, 0, sizeof(*im));
	err[0] = 0;
	if (len < 4 || p[0] != 0xFF || p[1] != 0xD8) { snprintf(err, 256, "not a JPEG file (no SOI)"); return -1; }
	pthread_once(&zz_mask_once, zz_mask_init);
	pv = (jq_priv*)calloc(1, sizeof(*pv));
	d = (jq_dec*)calloc(1, sizeof(*d));
	if (!pv || !d) { free(pv); free(d); snprintf(err, 256, "out of memory"); return -1; }
	im->priv = pv; d->im = im; d->pv = pv;
	pv->mem.pub.request_virt_barray = jq_request;
	pv->mem.pub.realize_virt_arrays = jq_realize;
	pv->mem.pub.access_virt_barray = jq_access;
	im->cinfo.mem = &pv->mem.pub;
	im->cinfo.comp_info = pv->comps;
	tail = &im->markers;
	p += 2;
	while (!done) {
		unsigned code, seglen; const unsigned char *seg;
		if (p < end && *p != 0xFF) im->warnings++;      /* libjpeg: JWRN_EXTRANEOUS_DATA */
		while (p < end && *p != 0xFF) p++;              /* tolerate garbage between segments */
		while (p < end && *p == 0xFF) p++;
		if (p >= end) { im->warnings++; break; }        /* no EOI: libjpeg's JWRN_JPEG_EOF */
		code = *p++;
		if (code == 0xD9) break;                        /* EOI */
		if (code == 0x01 || (code >= 0xD0 && code <= 0xD7) || code == 0) continue;
		if (p + 2 > end) break;
		seglen = be16(p);
		if (seglen < 2 || p + seglen > end) { snprintf(err, 256, "truncated marker segment 0x%02X", code); goto fail; }
		seg = p + 2; p += seglen; seglen -= 2;
		if (code == 0xDB) {                             /* DQT, B.2.4.1 */
			while (seglen >= 65) {
				int pq = seg[0] >> 4, tq = seg[0] & 15, n = pq ? 128 : 64;
				if (tq >= NUM_QUANT_TBLS || seglen < (unsigned)n + 1) { snprintf(err, 256, "bad DQT"); goto fail; }
				for (i = 0; i < 64; i++)
					pv->qt[tq].quantval[zz_nat[i]] = (UINT16)(pq ? be16(seg + 1 + 2 * i) : seg[1 + i]);
				im->cinfo.quant_tbl_ptrs[tq] = &pv->qt[tq];
				seg += n + 1; seglen -= n + 1;
			}
		} else if (code == 0xC4) {                      /* DHT, B.2.4.2 */
			while (seglen >= 17) {
				int tc = seg[0] >> 4, th = seg[0] & 15, n = 0;
				jq_dhuff *h;
				if (tc > 1 || th > 3) { snprintf(err, 256, "bad DHT"); goto fail; }
				h = tc ? &d->ac[th] : &d->dc[th];
				h->bits[0] = 0;
				for (i = 1; i <= 16; i++) { h->bits[i] = seg[i]; n += seg[i]; }
				if (n > 256 || seglen < 17u + n) { snprintf(err, 256, "bad DHT"); goto fail; }
				memcpy(h->val, seg + 17, n);
				if (dhuff_build(h)) { snprintf(err, 256, "bad Huffman table"); goto fail; }
				seg += 17 + n; seglen -= 17 + n;
			}
		} else if (code == 0xDD) {                      /* DRI */
			if (seglen >= 2) im->restart_interval = be16(seg);
		} else if (code == 0xC0 || code == 0xC1 || code == 0xC2) {      /* SOF0/1/2, B.2.2 */
			int nf, maxh = 1, maxv = 1;
			if (have_frame || seglen < 6) { snprintf(err, 256, "bad frame header"); goto fail; }
			if (seg[0] != 8) { snprintf(err, 256, "%d-bit samples are not supported", seg[0]); goto fail; }
			im->progressive = code == 0xC2;
			sof_code = (int)code;
			im->cinfo.image_height = be16(seg + 1); im->cinfo.image_width = be16(seg + 3);
			nf = seg[5];
			if (nf < 1 || nf > 4 || seglen < 6u + 3 * nf || !im->cinfo.image_width || !im->cinfo.image_height) {
				snprintf(err, 256, "unsupported frame header (%d components)", nf); goto fail;
			}
			im->cinfo.num_components = nf;
			for (i = 0; i < nf; i++) {
				jpeg_component_info *c = &pv->comps[i];
				im->comp_id[i] = seg[6 + 3 * i];
				c->component_id = seg[6 + 3 * i]; c->component_index = i;
				c->h_samp_factor = seg[7 + 3 * i] >> 4; c->v_samp_factor = seg[7 + 3 * i] & 15;
				c->quant_tbl_no = seg[8 + 3 * i] & 3;
				if (c->h_samp_factor < 1 || c->h_samp_factor > 4 || c->v_samp_factor < 1 || c->v_samp_factor > 4) {
					snprintf(err, 256, "bad sampling factors"); goto fail;
				}
				if (c->h_samp_factor > maxh) maxh = c->h_samp_factor;
				if (c->v_samp_factor > maxv) maxv = c->v_samp_factor;
			}
			im->cinfo.max_h_samp_factor = maxh; im->cinfo.max_v_samp_factor = maxv;
			d->mcux = (im->cinfo.image_width + 8 * maxh - 1) / (8 * maxh);
			d->mcuy = (im->cinfo.image_height + 8 * maxv - 1) / (8 * maxv);
			for (i = 0; i < nf; i++) {
				jpeg_component_info *c = &pv->comps[i];
				/* libjpeg geometry (jdinput.c initial_setup): not padded to the MCU */
				c->width_in_blocks = (im->cinfo.image_width * c->h_samp_factor + 8 * maxh - 1) / (8 * maxh);
				c->height_in_blocks = (im->cinfo.image_height * c->v_samp_factor + 8 * maxv - 1) / (8 * maxv);
				if (hdr || skip_data) continue;             /* header / markers only: no arrays */
				im->coef_arrays[i] = jq_request((j_common_ptr)&im->cinfo, JPOOL_IMAGE, TRUE,
						d->mcux * c->h_samp_factor, d->mcuy * c->v_samp_factor, 1);
				if (!im->coef_arrays[i]) { snprintf(err, 256, "out of memory"); goto fail; }
			}
			/* colour space guess of jdapimin.c default_decompress_parms (JFIF / Adobe aside) */
			im->cinfo.jpeg_color_space = nf == 1 ? JCS_GRAYSCALE : nf == 3 ? JCS_YCbCr : JCS_CMYK;
			if (nf == 3 && im->comp_id[0] == 'R' && im->comp_id[1] == 'G' && im->comp_id[2] == 'B')
				im->cinfo.jpeg_color_space = JCS_RGB;
			have_frame = 1;
		} else if (code >= 0xC3 && code <= 0xCF && code != 0xC8) {
			snprintf(err, 256, "unsupported JPEG process (SOF%d: lossless, hierarchical or arithmetic)", code - 0xC0);
			goto fail;
		} else if (code == 0xDA) {                      /* SOS, B.2.3 */
			jq_scan s; int ns;
			if (!have_frame || seglen < 1) { snprintf(err, 256, "SOS before SOF"); goto fail; }
			ns = seg[0];
			if (ns < 1 || ns > 4 || seglen < 4u + 2 * ns) { snprintf(err, 256, "bad scan header"); goto fail; }
			memset(&s, 0, sizeof(s)); s.ncomp = ns;
			for (i = 0; i < ns; i++) {
				int id = seg[1 + 2 * i], j;
				for (j = 0; j < im->cinfo.num_components && im->comp_id[j] != id; j++);
				if (j == im->cinfo.num_components) { snprintf(err, 256, "scan names an unknown component"); goto fail; }
				s.ci[i] = j; s.td[i] = (seg[2 + 2 * i] >> 4) & 3; s.ta[i] = seg[2 + 2 * i] & 3;
			}
			s.Ss = seg[1 + 2 * ns]; s.Se = seg[2 + 2 * ns]; s.Ah = seg[3 + 2 * ns] >> 4; s.Al = seg[3 + 2 * ns] & 15;
			if (!im->progressive) { s.Ss = 0; s.Se = 63; s.Ah = s.Al = 0; }
			if (s.Ss > s.Se || s.Se > 63 || s.Al > 13 || (s.Ss > 0 && ns != 1)) { snprintf(err, 256, "bad scan parameters"); goto fail; }
			d->ri = im->restart_interval;
			if (hdr) {                                  /* header only: stop before the entropy-coded data */
				memset(hdr, 0, sizeof(*hdr));
				hdr->sof = im->progressive ? 0xC2 : sof_code; hdr->ncomp = ns;
				for (i = 0; i < ns; i++) { hdr->ci[i] = s.ci[i]; hdr->td[i] = s.td[i]; hdr->ta[i] = s.ta[i]; }
				for (i = 0; i < 4; i++) {
					hdr->dc_present[i] = d->dc[i].present; hdr->ac_present[i] = d->ac[i].present;
					memcpy(hdr->dc_bits[i], d->dc[i].bits, 17); memcpy(hdr->dc_val[i], d->dc[i].val, 256);
					memcpy(hdr->ac_bits[i], d->ac[i].bits, 17); memcpy(hdr->ac_val[i], d->ac[i].val, 256);
				}
				hdr->restart_interval = im->restart_interval;
				hdr->entropy_offset = (size_t)(p - data);
				done = 1;
				continue;
			}
			if (skip_data) {                            /* markers only: on to the next marker, as defer does */
				if (rec && rec->n < rec->cap) {
					jq_scanrec *r = &rec->recs[rec->n];
					memset(r, 0, sizeof(*r));
					r->sof = im->progressive ? 0xC2 : sof_code;
					r->ncomp = ns; r->Ss = s.Ss; r->Se = s.Se; r->Ah = s.Ah; r->Al = s.Al;
					for (i = 0; i < ns; i++) { r->ci[i] = s.ci[i]; r->td[i] = s.td[i]; r->ta[i] = s.ta[i]; }
					for (i = 0; i < 4; i++) {
						r->dc_present[i] = d->dc[i].present; r->ac_present[i] = d->ac[i].present;
						memcpy(r->dc_bits[i], d->dc[i].bits, 17); memcpy(r->dc_val[i], d->dc[i].val, 256);
						memcpy(r->ac_bits[i], d->ac[i].bits, 17); memcpy(r->ac_val[i], d->ac[i].val, 256);
					}
					r->restart_interval = im->restart_interval;
					r->offset = (size_t)(p - data);
				}
				p = next_marker(p, end);
				if (rec) {
					/* the walk stops one byte short of the file's end when no marker follows (a file
					 * cut inside entropy-coded data): that last byte is part of the segment */
					if (rec->n < rec->cap) rec->recs[rec->n].end = p + 1 >= end ? len : (size_t)(p - data);
					rec->n++;
				}
				continue;
			}
			if (defer && im->progressive) {                 /* record the scan, find the next marker */
				const unsigned char *q = p; jq_dscan *c;
				if (ndsc == JQ_MAX_DEFER) { retry = 1; goto fail; }
				if (!dsc) dsc = (jq_dscan*)calloc(JQ_MAX_DEFER, sizeof(*dsc));
				c = dsc ? &dsc[ndsc] : NULL;
				if (!c || !(c->d = (jq_dec*)malloc(sizeof(*d)))) { retry = 1; goto fail; }
				ndsc++;
				memcpy(c->d, d, sizeof(*d)); c->d->warn = 0;
				c->s = s; c->p = p;
				while (q + 1 < end && !(q[0] == 0xFF && q[1] != 0 && q[1] != 0xFF && (q[1] & 0xF8) != 0xD0)) q++;
				c->segend = q; p = q;
				continue;
			}
			if (dec_scan(d, &s, p, end, &p, err)) goto fail;
			im->warnings += d->warn; d->warn = 0;
		} else if ((code >= 0xE0 && code <= 0xEF) || code == 0xFE) {
			int want = code == 0xFE ? copy > 0 : copy > 1;
			if (code == 0xEE && seglen >= 12 && !memcmp(seg, "Adobe", 5)) {       /* transform flag, jdmarker.c */
				adobe = seg[11];
				im->saw_adobe = 1; im->adobe_transform = seg[11];
			}
			if (code == 0xE0 && seglen >= 14 && !memcmp(seg, "JFIF", 5)) {         /* jdmarker.c examine_app0 */
				im->saw_jfif = 1; im->jfif_major = seg[5]; im->jfif_minor = seg[6];
				im->density_unit = seg[7]; im->x_density = (int)be16(seg + 8); im->y_density = (int)be16(seg + 10);
			}
			if (want) {
				jq_marker *m = (jq_marker*)calloc(1, sizeof(*m));
				if (!m || !(m->data = (unsigned char*)malloc(seglen + 1))) { free(m); snprintf(err, 256, "out of memory"); goto fail; }
				m->code = (int)code; m->len = seglen; memcpy(m->data, seg, seglen);
				*tail = m; tail = &m->next;
			}
		}
	}
	if (!have_frame) { snprintf(err, 256, "no frame header found"); goto fail; }
	if (ndsc && sched_run(im, dsc, ndsc, end)) { retry = 1; goto fail; }
	if (im->saw_jfif && im->cinfo.num_components == 3) im->cinfo.jpeg_color_space = JCS_YCbCr;
	if (adobe >= 0 && !(im->saw_jfif && im->cinfo.num_components == 3)) {      /* jdapimin.c default_decompress_parms */
		if (im->cinfo.num_components == 3) im->cinfo.jpeg_color_space = adobe == 0 ? JCS_RGB : JCS_YCbCr;
		/* 0: CMYK; 2 and every other value YCCK (libjpeg warns JWRN_ADOBE_XFORM for those, this reader does not) */
		if (im->cinfo.num_components == 4) im->cinfo.jpeg_color_space = adobe == 0 ? JCS_CMYK : JCS_YCCK;
	}
	for (i = 0; i < im->cinfo.num_components; i++) {
		jpeg_component_info *c = &pv->comps[i];
		c->quant_table = im->cinfo.quant_tbl_ptrs[c->quant_tbl_no];
		if (!c->quant_table) { snprintf(err, 256, "component %d uses an undefined quantization table", i); goto fail; }
	}
	for (i = 0; i < ndsc; i++) free(dsc[i].d);
	free(dsc); free(d);
	return 0;
fail:
	for (i = 0; i < ndsc; i++) free(dsc[i].d);
	free(dsc); free(d);
	jq_free(im);
	/* in deferred mode every failure is looked at again by the plain reader: it decides and words it */
	return retry || defer ? 1 : -1;
}

int jq_read(const unsigned char *data, size_t len, int copy, jq_image *im, char *err) {
	if (codec_thread_count() >= 2 && !getenv("JPEGQS_SERIAL_DECODE")) {
		int rc = jq_read_impl(data, len, copy, im, err, 1, NULL, 0, NULL);
		if (rc <= 0) return rc;
		if (getenv("JPEGQS_CODEC_TRACE")) fprintf(stderr, "jpegcoef: reading the file again, scan after scan\n");
	}
	return jq_read_impl(data, len, copy, im, err, 0, NULL, 0, NULL) ? -1 : 0;
}

int jq_read_header(const unsigned char *data, size_t len, jq_image *im, jq_header *hdr, char *err) {
	if (!hdr) { snprintf(err, 256, "no header record"); return -1; }
	memset(hdr, 0, sizeof(*hdr));
	if (jq_read_impl(data, len, 0, im, err, 0, hdr, 0, NULL)) return -1;
	if (!hdr->ncomp) { jq_free(im); snprintf(err, 256, "no scan found"); return -1; }
	return 0;
}

int jq_read_markers(const unsigned char *data, size_t len, int copy, jq_image *im, char *err) {
	return jq_read_impl(data, len, copy, im, err, 0, NULL, 1, NULL) ? -1 : 0;
}

int jq_read_scans(const unsigned char *data, size_t len, int copy, jq_image *im, jq_scanrec *recs, int cap, int *nrec, char *err) {
	jq_recs r; int rc;
	r.recs = recs; r.cap = recs ? cap : 0; r.n = 0;
	rc = jq_read_impl(data, len, copy, im, err, 0, NULL, 1, &r) ? -1 : 0;
	*nrec = r.n;
	return rc;
}

/* ---------------------------------------------------------------- the writer */
typedef struct { unsigned char *p; size_t n, cap; uint64_t acc; int nacc; int fail; } jq_out;

static void out_byte(jq_out *o, unsigned v) {
	if (o->n == o->cap) {
		size_t nc = o->cap ? o->cap * 2 : 1 << 16; unsigned char *q = (unsigned char*)realloc(o->p, nc);
		if (!q) { o->fail = 1; return; }
		o->p = q; o->cap = nc;
	}
	o->p[o->n++] = (unsigned char)v;
}
static void out_be16(jq_out *o, unsigned v) { out_byte(o, v >> 8); out_byte(o, v & 255); }
static void out_bits(jq_out *o, unsigned code, int n) {
	o->acc = (o->acc << n) | (code & ((1u << n) - 1)); o->nacc += n;
	while (o->nacc >= 8) {
		unsigned b = (unsigned)(o->acc >> (o->nacc - 8)) & 255;
		out_byte(o, b); if (b == 0xFF) out_byte(o, 0);
		o->nacc -= 8;
	}
}
static void out_flush(jq_out *o) { if (o->nacc) out_bits(o, 0x7F, 8 - o->nacc); o->acc = 0; o->nacc = 0; }

typedef struct {
	unsigned char bits[17], val[256]; int nval;
	unsigned code[256]; unsigned char size[256];
	uint32_t cs[256];                    /* (code << 8) | size: one load per symbol in the block coder */
	long freq[257];
} jq_ehuff;

/* T.81 K.3.3 example tables */
static const unsigned char std_dc_l_bits[17] = { 0, 0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0 };
static const unsigned char std_dc_c_bits[17] = { 0, 0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0 };
static const unsigned char std_dc_val[12] = { 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11 };
static const unsigned char std_ac_l_bits[17] = { 0, 0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d };
static const unsigned char std_ac_l_val[162] = {
	0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71,
	0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72,
	0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37,
	0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
	0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
	0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3,
	0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
	0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
	0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa };
static const unsigned char std_ac_c_bits[17] = { 0, 0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77 };
static const unsigned char std_ac_c_val[162] = {
	0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22,
	0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1,
	0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36,
	0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
	0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
	0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a,
	0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
	0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
	0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa };

static void ehuff_set(jq_ehuff *h, const unsigned char *bits, const unsigned char *val, int n) {
	memcpy(h->bits, bits, 17); memcpy(h->val, val, n); h->nval = n;
}
static void ehuff_codes(jq_ehuff *h) {                  /* T.81 C.2 */
	int l, i, k = 0; unsigned code = 0;
	memset(h->size, 0, sizeof(h->size));
	for (l = 1; l <= 16; l++) {
		for (i = 0; i < h->bits[l]; i++, k++) { h->code[h->val[k]] = code++; h->size[h->val[k]] = (unsigned char)l; }
		code <<= 1;
	}
	for (i = 0; i < 256; i++) h->cs[i] = h->size[i] ? (uint32_t)h->code[i] << 8 | h->size[i] : 0;
}
/* optimal code lengths limited to 16 bits, T.81 K.2 (figures K.1 - K.4) */
static void ehuff_optimal(jq_ehuff *h) {
	long freq[257]; int codesize[257], others[257], bits[33], i, j, c1, c2, k;
	memcpy(freq, h->freq, sizeof(freq));
	memset(codesize, 0, sizeof(codesize)); memset(bits, 0, sizeof(bits));
	for (i = 0; i < 257; i++) others[i] = -1;
	freq[256] = 1;                                       /* reserves the all-ones code */
	for (;;) {
		long v = 1000000000L;
		c1 = -1; c2 = -1;
		for (i = 0; i <= 256; i++) if (freq[i] && freq[i] <= v) { v = freq[i]; c1 = i; }
		v = 1000000000L;
		for (i = 0; i <= 256; i++) if (freq[i] && freq[i] <= v && i != c1) { v = freq[i]; c2 = i; }
		if (c2 < 0) break;
		freq[c1] += freq[c2]; freq[c2] = 0;
		for (codesize[c1]++; others[c1] >= 0; codesize[c1]++) c1 = others[c1];
		others[c1] = c2;
		for (codesize[c2]++; others[c2] >= 0; codesize[c2]++) c2 = others[c2];
	}
	for (i = 0; i <= 256; i++) if (codesize[i]) bits[codesize[i] > 32 ? 32 : codesize[i]]++;
	for (i = 32; i > 16; i--) while (bits[i] > 0) {
		for (j = i - 2; bits[j] == 0; j--);
		bits[i] -= 2; bits[i - 1]++; bits[j + 1] += 2; bits[j]--;
	}
	while (bits[i] == 0) i--;
	bits[i]--;                                           /* drop the reserved code point */
	memset(h->bits, 0, sizeof(h->bits));
	for (i = 1; i <= 16; i++) h->bits[i] = (unsigned char)bits[i];
	for (k = 0, i = 1; i <= 32; i++) for (j = 0; j < 256; j++) if (codesize[j] == i) h->val[k++] = (unsigned char)j;
	h->nval = k;
}

/* ---------------------------------------------------------------- entropy coding of the scan
 * The one interleaved scan is cut into segments of MCU rows that worker threads code
 * independently: a segment's DC predictors are the DC values of the last real blocks of the MCU
 * row above it (padding blocks repeat the predictor, so they never change it), and its bits go
 * to a private buffer WITHOUT byte stuffing.  The segments are then appended in order to the
 * output, shifted to the running bit position and stuffed there.  The result is byte for byte
 * what a sequential coder writes, whatever the number of threads. */
static int jq_threads_wanted = 0;
void jq_set_threads(int n) { jq_threads_wanted = n; }

static inline int bit_size(int v) { unsigned a = (unsigned)(v < 0 ? -v : v); return a ? 32 - __builtin_clz(a) : 0; }

typedef struct {
	unsigned char *p; size_t n, cap;     /* whole bytes, unstuffed */
	uint64_t acc; int nacc;              /* pending bits: < 32 after a block, < 8 after seg_finish */
	int fail;
	char pad[128];                       /* workers write neighbouring entries: keep them on separate cache lines */
} jq_seg;

typedef struct {
	jq_image *im; jvirt_barray_ptr *arrays;
	const jq_ehuff *dc, *ac;             /* NULL: count symbols only */
	JDIMENSION mcux, mcuy;
	int nseg; volatile int next;         /* dynamic segment queue */
	jq_seg *seg;                         /* [nseg] code bits */
	long (*freq)[4][257];                /* [nseg] dc0, ac0, dc1, ac1 symbol counts */
	volatile int range_error;
} jq_enc;

/* code bits go to a 64-bit accumulator that is emptied four bytes at a time: at most 31 bits are
 * pending before a put, a put adds at most 27 (a 16-bit code + 11 value bits) */
#define SEG_PUT(code, size) do { acc = (acc << (size)) | (uint64_t)(code); nacc += (size); \
	if (nacc >= 32) { uint32_t x_ = __builtin_bswap32((uint32_t)(acc >> (nacc - 32))); memcpy(w, &x_, 4); w += 4; nacc -= 32; } } while (0)

/* one block: counts symbols (sg == NULL) or appends its code bits to the segment */
static inline int enc_block(jq_seg *sg, const JCOEF *blk, int *pred, const jq_ehuff *dc, const jq_ehuff *ac,
		long *fdc, long *fac) {
	int diff = blk[0] - *pred, s = bit_size(diff), k, prev = 0, run;
	uint64_t zm = nonzero_mask_zz(blk) & ~1ULL;
	*pred = blk[0];
	if (s > 11) return -1;
	if (!sg) {
		fdc[s]++;
		while (zm) {
			k = __builtin_ctzll(zm); zm &= zm - 1;
			run = k - prev - 1; prev = k;
			for (; run > 15; run -= 16) fac[0xF0]++;
			s = bit_size(blk[zz_nat[k]]);
			if (s > 10) return -1;
			fac[run << 4 | s]++;
		}
		if (prev != 63) fac[0]++;
		return 0;
	}
	{
		uint64_t acc = sg->acc; int nacc = sg->nacc;
		unsigned char *w = sg->p + sg->n;            /* the caller reserved room for a whole block */
		uint32_t cs = dc->cs[s];
		SEG_PUT((uint64_t)(cs >> 8) << s | ((unsigned)(diff + (diff >> 31)) & ((1u << s) - 1)), (int)(cs & 255) + s);
		while (zm) {
			int v;
			k = __builtin_ctzll(zm); zm &= zm - 1;
			run = k - prev - 1; prev = k;
			v = blk[zz_nat[k]];
			for (; run > 15; run -= 16) SEG_PUT(ac->cs[0xF0] >> 8, (int)(ac->cs[0xF0] & 255));
			s = bit_size(v);
			if (s > 10) return -1;
			cs = ac->cs[run << 4 | s];
			/* value bits: v for v > 0, v - 1 for v < 0 (F.1.2.1), the low s bits of it */
			SEG_PUT((uint64_t)(cs >> 8) << s | ((unsigned)(v + (v >> 31)) & ((1u << s) - 1)), (int)(cs & 255) + s);
		}
		if (prev != 63) SEG_PUT(ac->cs[0] >> 8, (int)(ac->cs[0] & 255));
		sg->acc = acc; sg->nacc = nacc; sg->n = (size_t)(w - sg->p);
	}
	return 0;
}

/* whole bytes of the pending bits to the buffer: fewer than 8 stay (room: see enc_rows) */
static void seg_finish(jq_seg *sg) {
	while (sg->nacc >= 8) { sg->nacc -= 8; sg->p[sg->n++] = (unsigned char)(sg->acc >> sg->nacc); }
	sg->acc &= 0xFF;
}

/* MCU rows [y0, y1): walk = 1 only tracks the DC predictors (used for the row above a segment) */
static int enc_rows(jq_enc *e, JDIMENSION y0, JDIMENSION y1, int *pred, jq_seg *sg, long (*fr)[257], int walk) {
	struct jpeg_decompress_struct *ci = &e->im->cinfo;
	JDIMENSION x, y; int k, single = ci->num_components == 1;  /* one component: one block per MCU */
	static const JCOEF zero[64] = { 0 };
	for (y = y0; y < y1; y++) {
		JBLOCKROW rows[MAX_COMPONENTS][4];
		for (k = 0; k < ci->num_components; k++) {
			jpeg_component_info *c = &ci->comp_info[k]; int v, vf = single ? 1 : c->v_samp_factor;
			for (v = 0; v < vf && v < 4; v++) {
				JDIMENSION by = y * vf + v;
				rows[k][v] = by < c->height_in_blocks ?
						(*ci->mem->access_virt_barray)((j_common_ptr)ci, e->arrays[k], by, 1, FALSE)[0] : NULL;
			}
		}
		for (x = 0; x < e->mcux; x++) for (k = 0; k < ci->num_components; k++) {
			jpeg_component_info *c = &ci->comp_info[k]; int h, v, t = k ? 1 : 0;
			int hf = single ? 1 : c->h_samp_factor, vf = single ? 1 : c->v_samp_factor;
			for (v = 0; v < vf; v++) for (h = 0; h < hf; h++) {
				JDIMENSION bx = x * hf + h;
				JCOEF dummy[64];
				const JCOEF *blk;
				if (bx < c->width_in_blocks && rows[k][v]) blk = rows[k][v][bx];
				else if (walk) continue;                     /* padding keeps the predictor */
				else {                                       /* padding block: DC repeats, AC zero (like jctrans.c) */
					memcpy(dummy, zero, sizeof(dummy)); dummy[0] = (JCOEF)pred[k]; blk = dummy;
				}
				if (walk) { pred[k] = blk[0]; continue; }
				if (sg && sg->cap - sg->n < 512) {           /* a block is at most 1665 bits */
					size_t nc = sg->cap ? sg->cap * 2 : 1 << 16; unsigned char *q = (unsigned char*)realloc(sg->p, nc);
					if (!q) { sg->fail = 1; return -1; }
					sg->p = q; sg->cap = nc;
				}
				if (enc_block(sg, blk, &pred[k], e->dc ? &e->dc[t] : NULL, e->ac ? &e->ac[t] : NULL,
						fr ? fr[2 * t] : NULL, fr ? fr[2 * t + 1] : NULL)) return -1;
			}
		}
	}
	return 0;
}

static void *enc_worker(void *arg) {
	jq_enc *e = (jq_enc*)arg;
	for (;;) {
		int i = __sync_fetch_and_add(&e->next, 1), pred[MAX_COMPONENTS] = { 0 };
		JDIMENSION y0, y1;
		if (i >= e->nseg) break;
		y0 = (JDIMENSION)((uint64_t)e->mcuy * (unsigned)i / (unsigned)e->nseg);
		y1 = (JDIMENSION)((uint64_t)e->mcuy * (unsigned)(i + 1) / (unsigned)e->nseg);
		if (y0 > 0) enc_rows(e, y0 - 1, y0, pred, NULL, NULL, 1);
		if (enc_rows(e, y0, y1, pred, e->dc ? &e->seg[i] : NULL, e->dc ? NULL : e->freq[i], 0) &&
				!(e->dc && e->seg[i].fail)) e->range_error = 1;
		if (e->dc && e->seg[i].p) seg_finish(&e->seg[i]);
	}
	return NULL;
}

static int codec_thread_count(void) {
	int n = jq_threads_wanted;
	const char *env = getenv("JPEGQS_CODEC_THREADS");
	if (env && atoi(env) > 0) n = atoi(env);
	if (n <= 0) { long c = sysconf(_SC_NPROCESSORS_ONLN); n = c > 0 ? (int)c : 1; if (n > 16) n = 16; }
	if (n > 64) n = 64;
	return n < 1 ? 1 : n;
}
static int enc_thread_count(JDIMENSION mcuy) {
	int n = codec_thread_count();
	if ((JDIMENSION)n > mcuy) n = (int)mcuy;
	return n < 1 ? 1 : n;
}

/* appends a segment's bits at the output's current bit position, stuffing FF bytes.  Eight
 * bytes at a time: shifted to the output's bit phase, tested for an FF byte with one
 * arithmetic expression, stored whole when there is none. */
static void out_segment(jq_out *o, const jq_seg *sg) {
	size_t i = 0, need = o->n + 2 * sg->n + 32;
	int k = o->nacc;                                    /* 0..7 bits already pending in o->acc */
	if (need > o->cap) {
		size_t nc = o->cap ? o->cap : 1 << 16; unsigned char *q;
		while (nc < need) nc *= 2;
		q = (unsigned char*)realloc(o->p, nc);
		if (!q) { o->fail = 1; return; }
		o->p = q; o->cap = nc;
	}
	{
		unsigned char *w = o->p + o->n;
		uint64_t carry = k ? o->acc & ((1ULL << k) - 1) : 0;
		for (; i + 8 <= sg->n; i += 8) {
			uint64_t x, v; int j;
			memcpy(&x, sg->p + i, 8); x = __builtin_bswap64(x);      /* first byte on top */
			v = k ? carry << (64 - k) | x >> k : x;
			carry = x;                                               /* its low k bits are the new pending bits */
			if (!((~v - 0x0101010101010101ULL) & v & 0x8080808080808080ULL)) {
				uint64_t be = __builtin_bswap64(v); memcpy(w, &be, 8); w += 8;
			} else for (j = 56; j >= 0; j -= 8) {
				unsigned c = (unsigned)(v >> j) & 255;
				*w++ = (unsigned char)c; if (c == 0xFF) *w++ = 0;
			}
		}
		o->n = (size_t)(w - o->p);
		o->acc = k ? carry & ((1ULL << k) - 1) : 0;
	}
	for (; i < sg->n; i++) out_bits(o, sg->p[i], 8);
	if (sg->nacc) out_bits(o, (unsigned)sg->acc & ((1u << sg->nacc) - 1), sg->nacc);
}

/* The splice on the worker threads.  Once every segment is coded its position in the scan's bit
 * stream is known (S = bits of the segments before it).  Output byte j belongs to the segment that
 * holds its first bit; that segment's thread shifts its bits into byte phase, takes the few bits the
 * last byte needs from the next segment, stuffs FF bytes, all into a buffer of its own.  What is
 * left for one thread is copying those buffers one after the other.  The bits after the last
 * whole byte of the scan stay pending in the output's accumulator, as out_segment leaves them. */
typedef struct {
	jq_seg *seg; int nseg;
	uint64_t *start;                     /* [nseg + 1] bit position of each segment in the scan */
	unsigned char **buf; size_t *len;    /* [nseg] stuffed bytes of each segment */
	volatile int next, fail;
} jq_splice;

/* bit t (0 = first) .. t+7 of segment i followed by the segments after it; zero beyond the scan */
static unsigned splice_byte(const jq_splice *sp, int i, uint64_t t) {
	unsigned v = 0; int got = 0;
	while (got < 8 && i < sp->nseg) {
		const jq_seg *sg = &sp->seg[i]; uint64_t L = 8 * (uint64_t)sg->n + (unsigned)sg->nacc;
		if (t >= L) { t -= L; i++; continue; }
		{
			unsigned bit;
			if (t < 8 * (uint64_t)sg->n) bit = (sg->p[t >> 3] >> (7 - (t & 7))) & 1;
			else bit = (unsigned)(sg->acc >> (sg->nacc - 1 - (int)(t - 8 * (uint64_t)sg->n))) & 1;
			v = v << 1 | bit; got++; t++;
		}
	}
	return v << (8 - got);
}

static void splice_segment(jq_splice *sp, int i) {
	const jq_seg *sg = &sp->seg[i];
	uint64_t S = sp->start[i], E = sp->start[i + 1];
	uint64_t j0 = (S + 7) >> 3, j1 = i + 1 < sp->nseg ? (E + 7) >> 3 : E >> 3;     /* owned bytes [j0, j1) */
	size_t nout = j1 > j0 ? (size_t)(j1 - j0) : 0, b = 0;
	unsigned o = (unsigned)(8 * j0 - S);                 /* leading bits that belong to the byte before */
	unsigned char *w, *dst = (unsigned char*)malloc(2 * nout + 16);
	if (!dst) { sp->fail = 1; return; }
	w = dst;
	/* eight bytes at a time while nine source bytes are there */
	for (; b + 8 <= nout && b + 9 <= sg->n; b += 8) {
		uint64_t x, v; int j;
		memcpy(&x, sg->p + b, 8); x = __builtin_bswap64(x);
		v = o ? x << o | (uint64_t)(sg->p[b + 8] >> (8 - o)) : x;
		if (!((~v - 0x0101010101010101ULL) & v & 0x8080808080808080ULL)) {
			uint64_t be = __builtin_bswap64(v); memcpy(w, &be, 8); w += 8;
		} else for (j = 56; j >= 0; j -= 8) {
			unsigned c = (unsigned)(v >> j) & 255;
			*w++ = (unsigned char)c; if (c == 0xFF) *w++ = 0;
		}
	}
	for (; b < nout; b++) {                              /* the end of the segment, bit by bit */
		unsigned c = splice_byte(sp, i, 8 * (uint64_t)b + o);
		*w++ = (unsigned char)c; if (c == 0xFF) *w++ = 0;
	}
	sp->buf[i] = dst; sp->len[i] = (size_t)(w - dst);
}
static void *splice_worker(void *arg) {
	jq_splice *sp = (jq_splice*)arg;
	for (;;) {
		int i = __sync_fetch_and_add(&sp->next, 1);
		if (i >= sp->nseg) break;
		splice_segment(sp, i);
	}
	return NULL;
}

/* 0 = done, -1 = not applicable or out of memory (nothing written: the caller splices serially) */
static int out_segments_parallel(jq_out *o, jq_seg *seg, int nseg, int nthr) {
	jq_splice sp; pthread_t tid[64]; int i, started = 0, rc = -1; size_t total = 0; uint64_t bits;
	if (nseg < 2 || nthr < 2 || o->nacc) return -1;
	memset(&sp, 0, sizeof(sp));
	sp.seg = seg; sp.nseg = nseg;
	sp.start = (uint64_t*)calloc((size_t)nseg + 1, sizeof(uint64_t));
	sp.buf = (unsigned char**)calloc((size_t)nseg, sizeof(*sp.buf));
	sp.len = (size_t*)calloc((size_t)nseg, sizeof(size_t));
	if (!sp.start || !sp.buf || !sp.len) goto out;
	for (i = 0; i < nseg; i++) {
		uint64_t L = 8 * (uint64_t)seg[i].n + (unsigned)seg[i].nacc;
		if (L < 64) goto out;                            /* a byte must not span more than two segments */
		sp.start[i + 1] = sp.start[i] + L;
	}
	for (i = 1; i < nthr && i < 64; i++) { if (pthread_create(&tid[started], NULL, splice_worker, &sp)) break; started++; }
	splice_worker(&sp);
	for (i = 0; i < started; i++) pthread_join(tid[i], NULL);
	if (sp.fail) goto out;
	for (i = 0; i < nseg; i++) total += sp.len[i];
	if (o->cap - o->n < total + 16) {
		size_t nc = o->cap ? o->cap : 1 << 16; unsigned char *q;
		while (nc < o->n + total + 16) nc *= 2;
		q = (unsigned char*)realloc(o->p, nc);
		if (!q) goto out;
		o->p = q; o->cap = nc;
	}
	for (i = 0; i < nseg; i++) { memcpy(o->p + o->n, sp.buf[i], sp.len[i]); o->n += sp.len[i]; }
	bits = sp.start[nseg] & 7;                           /* after the last whole byte */
	o->nacc = (int)bits;
	o->acc = bits ? splice_byte(&sp, nseg - 1, sp.start[nseg] - sp.start[nseg - 1] - bits) >> (8 - bits) : 0;
	rc = 0;
out:
	if (sp.buf) for (i = 0; i < nseg; i++) free(sp.buf[i]);
	free(sp.start); free(sp.buf); free(sp.len);
	return rc;
}

/* counts symbols into dc/ac[].freq (o == NULL) or writes the entropy-coded segment to o */
static int enc_pass(jq_image *im, jvirt_barray_ptr *arrays, jq_out *o, jq_ehuff *dc, jq_ehuff *ac) {
	struct jpeg_decompress_struct *ci = &im->cinfo;
	int maxh = ci->max_h_samp_factor, maxv = ci->max_v_samp_factor, nthr, i, j, k, rc = -1;
	int trace = getenv("JPEGQS_CODEC_TRACE") != NULL; double t_start = 0, t_coded = 0;
	jq_enc e; pthread_t tid[64];
	memset(&e, 0, sizeof(e));
	e.im = im; e.arrays = arrays;
	e.mcux = (ci->image_width + 8 * maxh - 1) / (8 * maxh); e.mcuy = (ci->image_height + 8 * maxv - 1) / (8 * maxv);
	if (ci->num_components == 1) {                       /* not interleaved: one block per MCU (A.2.2) */
		e.mcux = ci->comp_info[0].width_in_blocks; e.mcuy = ci->comp_info[0].height_in_blocks;
	}
	if (!e.mcuy || !e.mcux) return 0;
	for (k = 0; k < ci->num_components; k++) if (ci->comp_info[k].v_samp_factor > 4) return -1;
	pthread_once(&zz_mask_once, zz_mask_init);
	t_start = trace ? trace_ms() : 0;
	nthr = enc_thread_count(e.mcuy);
	e.nseg = nthr == 1 ? 1 : nthr * 4;
	if ((JDIMENSION)e.nseg > e.mcuy) e.nseg = (int)e.mcuy;
	if (o) { e.dc = dc; e.ac = ac; e.seg = (jq_seg*)calloc((size_t)e.nseg, sizeof(jq_seg)); if (!e.seg) return -1; }
	else { e.freq = (long (*)[4][257])calloc((size_t)e.nseg, sizeof(*e.freq)); if (!e.freq) return -1; }
	for (i = 1; i < nthr; i++) if (pthread_create(&tid[i], NULL, enc_worker, &e)) break;
	nthr = i;                                            /* threads that really started (+ this one) */
	enc_worker(&e);
	for (i = 1; i < nthr; i++) pthread_join(tid[i], NULL);
	t_coded = trace ? trace_ms() : 0;
	if (!e.range_error) {
		rc = 0;
		if (o) {
			for (i = 0; i < e.nseg; i++) if (e.seg[i].fail) o->fail = 1;
			if (!o->fail && out_segments_parallel(o, e.seg, e.nseg, nthr))
				for (i = 0; i < e.nseg; i++) out_segment(o, &e.seg[i]);
			if (trace) fprintf(stderr, "jpegcoef: scan coded on %d threads in %.1f ms (%d segments), spliced in %.1f ms (%zu bytes)\n",
					nthr, t_coded - t_start, e.nseg, trace_ms() - t_coded, o->n);
		} else for (i = 0; i < e.nseg; i++) for (j = 0; j < 257; j++) {
			dc[0].freq[j] += e.freq[i][0][j]; ac[0].freq[j] += e.freq[i][1][j];
			dc[1].freq[j] += e.freq[i][2][j]; ac[1].freq[j] += e.freq[i][3][j];
		}
	}
	if (e.seg) { for (i = 0; i < e.nseg; i++) free(e.seg[i].p); free(e.seg); }
	free(e.freq);
	return rc;
}

static void out_dht(jq_out *o, int tc_th, const jq_ehuff *h) {
	int i;
	out_be16(o, 0xFFC4); out_be16(o, 2 + 1 + 16 + h->nval); out_byte(o, tc_th);
	for (i = 1; i <= 16; i++) out_byte(o, h->bits[i]);
	for (i = 0; i < h->nval; i++) out_byte(o, h->val[i]);
}

/* SOI, then what libjpeg writes for every output file, whatever -c says (jcmarker.c write_file_header
 * after jpeg_copy_critical_parameters -> jpeg_set_colorspace): a JFIF APP0 for grayscale / YCbCr with
 * the source's version (if 1.x or 2.x) and density, an Adobe APP14 carrying the colour transform for
 * RGB / CMYK / YCCK - without it a decoder would guess YCbCr / CMYK - and then the copied markers.
 * Depends on the input file only: everything after it (DQT on) on the coefficients. */
static void out_prefix(jq_out *o, const jq_image *im) {
	J_COLOR_SPACE cs = im->cinfo.jpeg_color_space;
	int jfif = cs == JCS_GRAYSCALE || cs == JCS_YCbCr, adobe = cs == JCS_RGB || cs == JCS_CMYK || cs == JCS_YCCK, i;
	const jq_marker *m;
	out_be16(o, 0xFFD8);
	if (jfif) {
		int major = 1, minor = 1, unit = 0, xd = 1, yd = 1;
		if (im->saw_jfif) {                              /* jctrans.c jpeg_copy_critical_parameters */
			if (im->jfif_major == 1 || im->jfif_major == 2) { major = im->jfif_major; minor = im->jfif_minor; }
			unit = im->density_unit; xd = im->x_density; yd = im->y_density;
		}
		out_be16(o, 0xFFE0); out_be16(o, 16);
		out_byte(o, 'J'); out_byte(o, 'F'); out_byte(o, 'I'); out_byte(o, 'F'); out_byte(o, 0);
		out_byte(o, (unsigned)major); out_byte(o, (unsigned)minor); out_byte(o, (unsigned)unit);
		out_be16(o, (unsigned)xd); out_be16(o, (unsigned)yd); out_byte(o, 0); out_byte(o, 0);
	}
	if (adobe) {
		out_be16(o, 0xFFEE); out_be16(o, 14);
		out_byte(o, 'A'); out_byte(o, 'd'); out_byte(o, 'o'); out_byte(o, 'b'); out_byte(o, 'e');
		out_be16(o, 100); out_be16(o, 0); out_be16(o, 0);
		out_byte(o, cs == JCS_YCCK ? 2u : 0u);           /* jcmarker.c emit_adobe_app14 (1 = YCbCr never gets here) */
	}
	for (m = im->markers; m; m = m->next) {              /* jcopy_markers_execute, quantsmooth.c:581-590 */
		if (jfif && m->code == 0xE0 && m->len >= 5 && !memcmp(m->data, "JFIF", 5)) continue;   /* written above */
		if (adobe && m->code == 0xEE && m->len >= 5 && !memcmp(m->data, "Adobe", 5)) continue;
		out_byte(o, 0xFF); out_byte(o, (unsigned)m->code); out_be16(o, (unsigned)m->len + 2);
		for (i = 0; i < (int)m->len; i++) out_byte(o, m->data[i]);
	}
}

int jq_prefix(const jq_image *im, unsigned char **out, size_t *outlen) {
	jq_out o;
	memset(&o, 0, sizeof(o));
	out_prefix(&o, im);
	if (o.fail) { free(o.p); return -1; }
	*out = o.p; *outlen = o.n;
	return 0;
}

int jq_write(jq_image *im, jvirt_barray_ptr *arrays, int optimize, unsigned char **out, size_t *outlen, char *err) {
	struct jpeg_decompress_struct *ci = &im->cinfo;
	jq_out o; jq_ehuff *dc, *ac; int i, k, nt = ci->num_components > 1 ? 2 : 1, blocks = 0, sof = 0xC0;
	unsigned written_q = 0;
	memset(&o, 0, sizeof(o)); err[0] = 0;
	dc = (jq_ehuff*)calloc(2, sizeof(*dc)); ac = (jq_ehuff*)calloc(2, sizeof(*ac));
	if (!dc || !ac) { free(dc); free(ac); snprintf(err, 256, "out of memory"); return -1; }
	for (k = 0; k < ci->num_components; k++) blocks += ci->comp_info[k].h_samp_factor * ci->comp_info[k].v_samp_factor;
	if (ci->num_components > 1 && blocks > 10) { snprintf(err, 256, "more than 10 blocks per MCU: not written as one interleaved scan"); goto fail; }
	if (optimize) {
		if (enc_pass(im, arrays, NULL, dc, ac)) { snprintf(err, 256, "coefficient out of range for Huffman coding"); goto fail; }
		for (i = 0; i < nt; i++) { ehuff_optimal(&dc[i]); ehuff_optimal(&ac[i]); }
	} else {
		ehuff_set(&dc[0], std_dc_l_bits, std_dc_val, 12); ehuff_set(&ac[0], std_ac_l_bits, std_ac_l_val, 162);
		ehuff_set(&dc[1], std_dc_c_bits, std_dc_val, 12); ehuff_set(&ac[1], std_ac_c_bits, std_ac_c_val, 162);
	}
	for (i = 0; i < nt; i++) { ehuff_codes(&dc[i]); ehuff_codes(&ac[i]); }

	out_prefix(&o, im);
	for (k = 0; k < ci->num_components; k++) {           /* DQT for every table in use */
		int tq = ci->comp_info[k].quant_tbl_no & 3, prec = 0;
		JQUANT_TBL *t = ci->comp_info[k].quant_table ? ci->comp_info[k].quant_table : ci->quant_tbl_ptrs[tq];
		if (!t || (written_q >> tq & 1)) continue;
		written_q |= 1u << tq;
		for (i = 0; i < 64; i++) if (t->quantval[i] > 255) prec = 1;
		if (prec) sof = 0xC1;
		out_be16(&o, 0xFFDB); out_be16(&o, 2 + 1 + (prec ? 128 : 64)); out_byte(&o, (unsigned)(prec << 4 | tq));
		for (i = 0; i < 64; i++) { unsigned v = t->quantval[zz_nat[i]]; if (prec) out_be16(&o, v); else out_byte(&o, v); }
	}
	out_be16(&o, 0xFF00 | sof); out_be16(&o, 8 + 3 * ci->num_components); out_byte(&o, 8);
	out_be16(&o, ci->image_height); out_be16(&o, ci->image_width); out_byte(&o, ci->num_components);
	for (k = 0; k < ci->num_components; k++) {
		jpeg_component_info *c = &ci->comp_info[k];
		out_byte(&o, (unsigned)im->comp_id[k]); out_byte(&o, (unsigned)(c->h_samp_factor << 4 | c->v_samp_factor));
		out_byte(&o, (unsigned)c->quant_tbl_no);
	}
	for (i = 0; i < nt; i++) { out_dht(&o, i, &dc[i]); out_dht(&o, 0x10 | i, &ac[i]); }
	out_be16(&o, 0xFFDA); out_be16(&o, 6 + 2 * ci->num_components); out_byte(&o, ci->num_components);
	for (k = 0; k < ci->num_components; k++) { out_byte(&o, (unsigned)im->comp_id[k]); out_byte(&o, k ? 0x11 : 0x00); }
	out_byte(&o, 0); out_byte(&o, 63); out_byte(&o, 0);
	if (enc_pass(im, arrays, &o, dc, ac)) { snprintf(err, 256, "coefficient out of range for Huffman coding"); goto fail; }
	out_flush(&o);
	out_be16(&o, 0xFFD9);
	if (o.fail) { snprintf(err, 256, "out of memory"); goto fail; }
	free(dc); free(ac);
	*out = o.p; *outlen = o.n;
	return 0;
fail:
	free(dc); free(ac); free(o.p);
	return -1;
}
