/*
 * jpeg_io.c - the host side of reading JPEG files into the library's layout
 * (include/jpegqs_cuda.h "JPEG files to quantized coefficients"): the header parse that feeds
 * jpegqs_cuda_decode_async, and the host decode for the files the device decoder does not take.
 * Both use jpegcoef.c's reader; nothing here parses markers itself.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "jpegcoef.h"
#include "jpegqs_cuda.h"

void qs_set_host_error(const char *msg);          /* qs_cuda.cu: jpegqs_cuda_last_error(NULL) */

/* libjpeg's rule for a table it decodes with (jdhuff.c jpeg_make_d_derived_tbl): no all-ones code,
 * DC symbols <= 15.  jpegcoef.c is more lenient; the device decoder relies on it. */
static int table_ok(const unsigned char *bits, const unsigned char *val, int dc) {
	int l, i, k = 0; long code = 0;
	for (l = 1; l <= 16; l++) {
		for (i = 0; i < bits[l]; i++, k++, code++) if (k >= 256 || (dc && val[k] > 15)) return 0;
		if (code >= (1L << l)) return 0;
		code <<= 1;
	}
	return 1;
}

static void fill_image(const jq_image *im, jpegqs_cuda_image *img) {
	int c, k;
	memset(img, 0, sizeof(*img));
	img->ncomp = im->cinfo.num_components;
	img->is_ycbcr = im->cinfo.jpeg_color_space == JCS_YCbCr;
	img->image_width = im->cinfo.image_width; img->image_height = im->cinfo.image_height;
	for (c = 0; c < img->ncomp; c++) {
		const jpeg_component_info *ci = &im->cinfo.comp_info[c];
		jpegqs_cuda_comp *o = &img->comp[c];
		o->wblk = ci->width_in_blocks; o->hblk = ci->height_in_blocks;
		o->h_samp = ci->h_samp_factor; o->v_samp = ci->v_samp_factor;
		o->has_qtbl = ci->quant_table != NULL;
		if (ci->quant_table) for (k = 0; k < 64; k++) o->quant[k] = ci->quant_table->quantval[k];
	}
}

/* jpegqs_cuda_jpeg_parse's rule for the first scan (the same fields in jq_header and jq_scanrec): not
 * progressive, all frame components, at least one entropy-coded byte, tables libjpeg decodes with */
#define FIRST_SCAN_OK(h, nframe, offset, len) first_scan_ok((h).sof, (h).ncomp, nframe, offset, len, (h).td, (h).ta, \
		(h).dc_present, (h).ac_present, (h).dc_bits, (h).dc_val, (h).ac_bits, (h).ac_val)
static int first_scan_ok(int sof, int ncomp, int nframe, size_t offset, size_t len, const int *td, const int *ta,
		const int *dcp, const int *acp, unsigned char (*dcb)[17], unsigned char (*dcv)[256],
		unsigned char (*acb)[17], unsigned char (*acv)[256]) {
	int k, ok = sof != 0xC2 && ncomp == nframe && offset < len;
	for (k = 0; ok && k < ncomp; k++)
		ok = dcp[td[k]] && acp[ta[k]] && table_ok(dcb[td[k]], dcv[td[k]], 1) && table_ok(acb[ta[k]], acv[ta[k]], 0);
	return ok;
}

int jpegqs_cuda_jpeg_parse(const uint8_t *data, size_t len, jpegqs_cuda_image *img, jpegqs_cuda_scan *scan) {
	jq_image im; jq_header h; char err[256]; int k;
	if (!data || !img || !scan) { qs_set_host_error("jpegqs_cuda_jpeg_parse: NULL argument"); return JPEGQS_ERR_ARG; }
	if (jq_read_header(data, len, &im, &h, err)) { qs_set_host_error(err); return JPEGQS_ERR_ARG; }
	fill_image(&im, img);
	memset(scan, 0, sizeof(*scan));
	scan->ncomp = h.ncomp;
	for (k = 0; k < 4; k++) {
		scan->comp[k] = h.ci[k]; scan->dc_tbl[k] = h.td[k]; scan->ac_tbl[k] = h.ta[k];
		scan->dc_present[k] = h.dc_present[k]; scan->ac_present[k] = h.ac_present[k];
		memcpy(scan->dc_bits[k], h.dc_bits[k], 17); memcpy(scan->dc_val[k], h.dc_val[k], 256);
		memcpy(scan->ac_bits[k], h.ac_bits[k], 17); memcpy(scan->ac_val[k], h.ac_val[k], 256);
	}
	scan->restart_interval = (uint32_t)h.restart_interval;
	scan->entropy_offset = h.entropy_offset;
	scan->jpeg_color_space = (int32_t)im.cinfo.jpeg_color_space;
	scan->sof = h.sof;
	jq_free(&im);
	if (!FIRST_SCAN_OK(h, img->ncomp, h.entropy_offset, len)) {
		qs_set_host_error("jpegqs_cuda_jpeg_parse: only the host reader takes this file"); return JPEGQS_ERR_UNSUPPORTED;
	}
	return 0;
}

/* the coefficients a scan codes, as a zig-zag band: a progressive DC scan codes coefficient 0 only */
static void scan_band(const jq_scanrec *r, int prog, int *lo, int *hi) {
	*lo = r->Ss; *hi = prog && r->Ss == 0 ? 0 : r->Se;
}

/* jpegqs_cuda_jpeg_parse_scans' verdict on the recorded scans (n >= 1): 0, JPEGQS_ERR_UNSUPPORTED or
 * JPEGQS_ERR_ARG, with the reason in *why */
static int scans_check(const jq_scanrec *rec, int n, int prog, const char **why) {
	int i, j, k, unsupported = 0;
	*why = "only the host reader takes this file";
	if (n > JPEGQS_MAX_SCANS) { *why = "more than 64 scans"; unsupported = 1; }
	for (i = 0; i < n && i < JPEGQS_MAX_SCANS; i++) {
		const jq_scanrec *r = &rec[i];
		int need_dc = !prog || (r->Ss == 0 && r->Ah == 0), need_ac = prog ? r->Ss > 0 : 1, lo, hi;
		if (r->offset >= r->end) { *why = "a scan without entropy-coded data"; unsupported = 1; }      /* a file cut at this SOS */
		for (k = 0; k < r->ncomp; k++) {
			if ((need_dc && !r->dc_present[r->td[k]]) || (need_ac && !r->ac_present[r->ta[k]])) {
				*why = "scan uses an undefined Huffman table"; return JPEGQS_ERR_ARG;
			}
			if ((need_dc && !table_ok(r->dc_bits[r->td[k]], r->dc_val[r->td[k]], 1)) ||
					(need_ac && !table_ok(r->ac_bits[r->ta[k]], r->ac_val[r->ta[k]], 0))) { *why = "a Huffman table libjpeg rejects"; unsupported = 1; }
		}
		/* first scans (Ah = 0) of a component must code disjoint bands, and come before the
		 * refinement scans of their band: the device runs all first scans before any refinement */
		scan_band(r, prog, &lo, &hi);
		for (j = 0; j < i && r->Ah == 0; j++) {
			const jq_scanrec *e = &rec[j]; int elo, ehi, share = 0, a, b;
			for (a = 0; a < r->ncomp; a++) for (b = 0; b < e->ncomp; b++) share |= r->ci[a] == e->ci[b];
			scan_band(e, prog, &elo, &ehi);
			if (share && lo <= ehi && elo <= hi) { *why = "overlapping first scans"; unsupported = 1; }
		}
	}
	return unsupported ? JPEGQS_ERR_UNSUPPORTED : 0;
}

static void copy_rec(const jq_scanrec *r, jpegqs_cuda_scan_rec *o) {
	int k;
	memset(o, 0, sizeof(*o));
	o->ncomp = r->ncomp;
	for (k = 0; k < 4; k++) {
		o->comp[k] = r->ci[k]; o->dc_tbl[k] = r->td[k]; o->ac_tbl[k] = r->ta[k];
		o->dc_present[k] = r->dc_present[k]; o->ac_present[k] = r->ac_present[k];
		memcpy(o->dc_bits[k], r->dc_bits[k], 17); memcpy(o->dc_val[k], r->dc_val[k], 256);
		memcpy(o->ac_bits[k], r->ac_bits[k], 17); memcpy(o->ac_val[k], r->ac_val[k], 256);
	}
	o->Ss = r->Ss; o->Se = r->Se; o->Ah = r->Ah; o->Al = r->Al; o->sof = r->sof;
	o->restart_interval = (uint32_t)r->restart_interval;
	o->offset = r->offset; o->end = r->end;
}

int jpegqs_cuda_jpeg_parse_scans(const uint8_t *data, size_t len, jpegqs_cuda_image *img,
		jpegqs_cuda_scan_rec *scans, int cap, int *nscans) {
	jq_image im; char err[256]; int n = 0, i, prog, rc;
	jq_scanrec *rec; const char *why;
	if (!data || !img || !nscans || cap < 0 || (cap && !scans)) { qs_set_host_error("jpegqs_cuda_jpeg_parse_scans: NULL argument"); return JPEGQS_ERR_ARG; }
	rec = (jq_scanrec*)calloc(JPEGQS_MAX_SCANS, sizeof(*rec));
	if (!rec) { qs_set_host_error("jpegqs_cuda_jpeg_parse_scans: out of memory"); return JPEGQS_ERR_ARG; }
	if (jq_read_scans(data, len, 0, &im, rec, JPEGQS_MAX_SCANS, &n, err)) { free(rec); qs_set_host_error(err); return JPEGQS_ERR_ARG; }
	fill_image(&im, img);
	prog = im.progressive;
	jq_free(&im);
	*nscans = n;
	if (!n) { free(rec); qs_set_host_error("jpegqs_cuda_jpeg_parse_scans: no scan found"); return JPEGQS_ERR_ARG; }
	rc = scans_check(rec, n, prog, &why);
	if (rc == JPEGQS_ERR_ARG) { free(rec); qs_set_host_error("jpegqs_cuda_jpeg_parse_scans: scan uses an undefined Huffman table"); return rc; }
	if (n > cap) rc = JPEGQS_ERR_UNSUPPORTED;
	for (i = 0; i < n && i < cap && i < JPEGQS_MAX_SCANS; i++) copy_rec(&rec[i], &scans[i]);
	free(rec);
	if (rc) { qs_set_host_error("jpegqs_cuda_jpeg_parse_scans: only the host reader takes this file"); return JPEGQS_ERR_UNSUPPORTED; }
	return 0;
}

/* The route of a file through a transcode: jpegqs_cuda_transcode_route's rule, and what
 * jpegqs_cuda_transcode needs of a DEVICE file, from one markers-only walk.  Every output but reason
 * may be NULL.  On DEVICE and HOST: img filled (coef pointers NULL).  On DEVICE: *nscans = 0 and *scan filled when
 * decode_async takes the file, else recs[0 .. *nscans) for decode_scans_async; head->comp_id /
 * quant_tbl filled and *prefix (malloc'd, copy level `copy`) / *prefix_len set.  Writes no error
 * state, so any thread may call it. */
int qs_route_plan(const uint8_t *data, size_t len, int copy, jpegqs_cuda_file_info *info, jpegqs_cuda_image *img,
		jpegqs_cuda_scan *scan, jpegqs_cuda_scan_rec *recs, int *nscans, jpegqs_cuda_jpeg_head *head,
		uint8_t **prefix, size_t *prefix_len, const char **reason) {
	jq_image im; char err[256]; jq_scanrec *rec; int n = 0, i, k, nc, blocks = 0, seq, route = JPEGQS_ROUTE_HOST;
	const char *why = "", *check_why;
	if (prefix) *prefix = NULL;
	if (!data) { *reason = "no data"; return JPEGQS_ERR_ARG; }
	rec = (jq_scanrec*)calloc(JPEGQS_MAX_SCANS, sizeof(*rec));
	if (!rec) { *reason = "out of memory"; return JPEGQS_ERR_ARG; }
	if (jq_read_scans(data, len, copy, &im, rec, JPEGQS_MAX_SCANS, &n, err)) { free(rec); *reason = "the reader rejects the file"; return JPEGQS_ERR_ARG; }
	nc = im.cinfo.num_components;
	for (i = 0; i < nc; i++) blocks += im.cinfo.comp_info[i].h_samp_factor * im.cinfo.comp_info[i].v_samp_factor;
	if (info) {
		info->image_width = im.cinfo.image_width; info->image_height = im.cinfo.image_height;
		info->ncomp = nc; info->progressive = im.progressive; info->restart_interval = im.restart_interval;
	}
	/* the sequential decoder decodes the first scan only: a second scan would be lost */
	seq = n == 1 && FIRST_SCAN_OK(rec[0], nc, rec[0].offset, len);
	if (!n) why = "no scan";
	else if (im.warnings) why = "marker-level damage (extraneous bytes or no EOI)";
	else if (nc > 4) why = "more than 4 components";
	else if (nc > 1 && blocks > 10) why = "more than 10 blocks per MCU";
	else if (!seq && scans_check(rec, n, im.progressive, &check_why)) why = check_why;
	else {
		for (i = 0; i < n && i < JPEGQS_MAX_SCANS && !why[0]; i++)
			if (im.progressive && rec[i].Ss > 0 && rec[i].Ah > 0 && !rec[i].restart_interval)
				why = "progressive AC refinement scan without restart markers";
		if (!why[0]) { route = JPEGQS_ROUTE_DEVICE; why = seq ? "sequential, one scan" : im.progressive ? "progressive" : "several scans"; }
	}
	if (img) fill_image(&im, img);
	/* every route: the header's colour space, which the pixel path's colour modes read */
	if (scan) scan->jpeg_color_space = (int32_t)im.cinfo.jpeg_color_space;
	if (route == JPEGQS_ROUTE_DEVICE) {
		if (nscans) *nscans = seq ? 0 : n;
		if (scan && seq) {
			const jq_scanrec *r = &rec[0];
			memset(scan, 0, sizeof(*scan));
			scan->ncomp = r->ncomp;
			for (k = 0; k < 4; k++) {
				scan->comp[k] = r->ci[k]; scan->dc_tbl[k] = r->td[k]; scan->ac_tbl[k] = r->ta[k];
				scan->dc_present[k] = r->dc_present[k]; scan->ac_present[k] = r->ac_present[k];
				memcpy(scan->dc_bits[k], r->dc_bits[k], 17); memcpy(scan->dc_val[k], r->dc_val[k], 256);
				memcpy(scan->ac_bits[k], r->ac_bits[k], 17); memcpy(scan->ac_val[k], r->ac_val[k], 256);
			}
			scan->restart_interval = (uint32_t)r->restart_interval;
			scan->entropy_offset = r->offset;
			scan->jpeg_color_space = (int32_t)im.cinfo.jpeg_color_space;
			scan->sof = r->sof;
		}
		if (recs && !seq) for (i = 0; i < n; i++) copy_rec(&rec[i], &recs[i]);
		if (head) for (k = 0; k < 4; k++) {
			head->comp_id[k] = k < nc ? im.comp_id[k] : 0;
			head->quant_tbl[k] = k < nc ? im.cinfo.comp_info[k].quant_tbl_no : 0;
		}
		if (prefix && jq_prefix(&im, prefix, prefix_len)) { *prefix = NULL; route = JPEGQS_ERR_ARG; why = "out of memory"; }
	}
	jq_free(&im);
	free(rec);
	*reason = why;
	return route;
}

int jpegqs_cuda_transcode_route(const uint8_t *data, size_t len, const char **reason, jpegqs_cuda_file_info *info) {
	const char *why;
	int rc = qs_route_plan(data, len, 0, info, NULL, NULL, NULL, NULL, NULL, NULL, NULL, &why);
	if (reason) *reason = why;
	return rc;
}

int jpegqs_cuda_jpeg_read(const uint8_t *data, size_t len, const jpegqs_cuda_image *img) {
	jq_image im; char err[256]; int c, warn; JDIMENSION y;
	if (!data || !img) { qs_set_host_error("jpegqs_cuda_jpeg_read: NULL argument"); return JPEGQS_ERR_ARG; }
	if (jq_read(data, len, 0, &im, err)) { qs_set_host_error(err); return JPEGQS_ERR_ARG; }
	if (img->ncomp != im.cinfo.num_components) goto geometry;
	for (c = 0; c < img->ncomp; c++) {
		const jpeg_component_info *ci = &im.cinfo.comp_info[c];
		if (!img->comp[c].coef || img->comp[c].wblk != ci->width_in_blocks || img->comp[c].hblk != ci->height_in_blocks)
			goto geometry;
	}
	for (c = 0; c < img->ncomp; c++) {
		const jpegqs_cuda_comp *o = &img->comp[c];
		JBLOCKARRAY rows = im.cinfo.mem->access_virt_barray((j_common_ptr)&im.cinfo, im.coef_arrays[c], 0, o->hblk, FALSE);
		for (y = 0; y < o->hblk; y++) memcpy(o->coef + (size_t)y * o->wblk * 64, rows[y], (size_t)o->wblk * sizeof(JBLOCK));
	}
	warn = im.warnings;
	jq_free(&im);
	return warn;
geometry:
	jq_free(&im);
	qs_set_host_error("jpegqs_cuda_jpeg_read: the arrays do not match the file's geometry (or a coef is NULL)");
	return JPEGQS_ERR_ARG;
}

int jpegqs_cuda_jpeg_prefix(const uint8_t *data, size_t len, int copy, uint8_t *out, size_t cap, size_t *out_len,
		int32_t *ncomp, int32_t comp_id[4], int32_t quant_tbl[4]) {
	jq_image im; char err[256]; unsigned char *p = NULL; size_t n = 0; int k;
	if (!data || !out_len || !ncomp || !comp_id || !quant_tbl) { qs_set_host_error("jpegqs_cuda_jpeg_prefix: NULL argument"); return JPEGQS_ERR_ARG; }
	if (copy < 0 || copy > 2) { qs_set_host_error("jpegqs_cuda_jpeg_prefix: copy level outside 0..2"); return JPEGQS_ERR_ARG; }
	if (jq_read_markers(data, len, copy, &im, err)) { qs_set_host_error(err); return JPEGQS_ERR_ARG; }
	if (jq_prefix(&im, &p, &n)) { jq_free(&im); qs_set_host_error("jpegqs_cuda_jpeg_prefix: out of memory"); return JPEGQS_ERR_ARG; }
	*out_len = n;
	*ncomp = im.cinfo.num_components;
	for (k = 0; k < 4; k++) {
		int have = k < im.cinfo.num_components;
		comp_id[k] = have ? im.comp_id[k] : 0;
		quant_tbl[k] = have ? im.cinfo.comp_info[k].quant_tbl_no : 0;
	}
	jq_free(&im);
	if (out && cap >= n) memcpy(out, p, n);
	free(p);
	if (out && cap < n) { qs_set_host_error("jpegqs_cuda_jpeg_prefix: the prefix does not fit out (*out_len holds its size)"); return JPEGQS_ERR_ARG; }
	return 0;
}

/* ------------------------------------------------------------------------------------------
 * EXIF orientation (include/jpegqs_cuda.h jpegqs_cuda_jpeg_orientation): the transform Pillow's
 * ImageOps.exif_transpose applies after Image.open, restated from what Pillow does with the bytes,
 * not from the EXIF specification.  Every read stays inside the segment it belongs to.
 * ------------------------------------------------------------------------------------------ */
#define EXIF_RAISES (-1)      /* Pillow's getexif raises: no transform, and no XMP fallback */
#define EXIF_NO_TAG 0         /* no 0x0112 entry: the XMP packet decides */

static uint32_t exif_u16(const uint8_t *p, int be) { return be ? (uint32_t)p[0] << 8 | p[1] : (uint32_t)p[1] << 8 | p[0]; }
static uint32_t exif_u32(const uint8_t *p, int be) {
	return be ? (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]
	          : (uint32_t)p[3] << 24 | (uint32_t)p[2] << 16 | (uint32_t)p[1] << 8 | p[0];
}

/* bytes per value of each TIFF type Pillow loads (TiffImagePlugin's _load_dispatch); 0: skipped */
static int exif_unit(uint32_t typ) {
	static const unsigned char unit[17] = {0, 1, 1, 2, 4, 8, 1, 1, 2, 4, 8, 4, 8, 4, 0, 0, 8};
	return typ < 17 ? unit[typ] : 0;
}

/* 2..8 when the first value of an entry of type typ, as Pillow decodes it, equals that integer in a
 * Python dict lookup; 1 otherwise (bytes, str, NaN, other numbers) */
static int exif_value(uint32_t typ, const uint8_t *v, int be) {
	int64_t k = 0;
	switch (typ) {
	case 3: k = exif_u16(v, be); break;                               /* SHORT */
	case 4: case 13: k = exif_u32(v, be); break;                      /* LONG, IFD */
	case 6: k = (int8_t)v[0]; break;                                  /* SIGNED BYTE */
	case 8: k = (int16_t)exif_u16(v, be); break;                      /* SIGNED SHORT */
	case 9: k = (int32_t)exif_u32(v, be); break;                      /* SIGNED LONG */
	case 16: {                                                        /* LONG8 */
		uint64_t hi = exif_u32(v + (be ? 0 : 4), be), lo = exif_u32(v + (be ? 4 : 0), be);
		k = hi ? 0 : (int64_t)lo; break;
	}
	case 5: case 10: {                                                /* (SIGNED) RATIONAL: a Fraction */
		uint32_t a = exif_u32(v, be), b = exif_u32(v + 4, be);
		int64_t num = typ == 5 ? (int64_t)a : (int64_t)(int32_t)a, den = typ == 5 ? (int64_t)b : (int64_t)(int32_t)b;
		k = den != 0 && num % den == 0 ? num / den : 0; break;
	}
	case 11: case 12: {                                               /* FLOAT, DOUBLE */
		double d;
		if (typ == 11) { uint32_t u = exif_u32(v, be); float f; memcpy(&f, &u, 4); d = f; }
		else { uint64_t u = (uint64_t)exif_u32(v + (be ? 0 : 4), be) << 32 | exif_u32(v + (be ? 4 : 0), be); memcpy(&d, &u, 8); }
		k = d >= 2 && d <= 8 && d == (double)(int)d ? (int)d : 0; break;
	}
	default: return 1;                                                /* BYTE, ASCII, UNDEFINED */
	}
	return k >= 2 && k <= 8 ? (int)k : 1;
}

/* Image.Exif.load and ImageFileDirectory_v2.load on the EXIF bytes d[0 .. n) (the first block without,
 * the later ones with their "Exif\0\0" stripped): EXIF_RAISES, EXIF_NO_TAG, or 1..8 from the last 0x0112
 * entry of IFD0 that Pillow keeps */
static int exif_ifd0_orientation(const uint8_t *d, size_t n) {
	size_t p, i, count; int be, found = EXIF_NO_TAG;
	while (n >= 6 && !memcmp(d, "Exif\0\0", 6)) { d += 6; n -= 6; }
	if (!n) return EXIF_NO_TAG;
	/* the TIFF header: byte order, 42 (or the swapped 42 Pillow also accepts); a BigTIFF header (43)
	 * raises, as does one shorter than 8 bytes */
	if (n < 4 || (memcmp(d, "MM\0*", 4) && memcmp(d, "II*\0", 4) && memcmp(d, "MM*\0", 4) && memcmp(d, "II\0*", 4)))
		return EXIF_RAISES;
	if (n < 8) return EXIF_RAISES;
	be = d[0] == 'M';
	p = exif_u32(d + 4, be);
	if (p > n || n - p < 2) return EXIF_NO_TAG;       /* the entry count cannot be read: an empty IFD */
	count = exif_u16(d + p, be);
	p += 2;
	for (i = 0; i < count; i++, p += 12) {
		uint32_t tag, typ; uint64_t size; const uint8_t *v;
		if (n - p < 12) break;                         /* a cut entry ends the IFD, keeping what was read */
		tag = exif_u16(d + p, be); typ = exif_u16(d + p + 2, be);
		if (!exif_unit(typ)) continue;                 /* a type Pillow does not load */
		size = (uint64_t)exif_u32(d + p + 4, be) * (uint64_t)exif_unit(typ);
		v = d + p + 8;
		if (size > 4) {
			uint32_t off = exif_u32(d + p + 8, be);
			if (off > n || n - off < size) break;          /* a read past the data ends the IFD */
			v = d + off;
		}
		if (!size) continue;                           /* an entry without data is not kept */
		if (tag == 0x0112) found = exif_value(typ, v, be);
	}
	return found;
}

/* the first decimal digit of the first "tiff:Orientation=\"" or "tiff:Orientation>" directly followed
 * by one (Pillow's regular expression), as the orientation; 1 if none */
static int xmp_orientation(const uint8_t *x, size_t n) {
	static const char key[] = "tiff:Orientation";
	const size_t k = sizeof(key) - 1;
	size_t i;
	for (i = 0; i + k < n; i++) {
		size_t j = i + k;
		if (memcmp(x + i, key, k)) continue;
		if (x[j] == '=' && j + 2 < n && x[j + 1] == '"' && x[j + 2] >= '0' && x[j + 2] <= '9') j += 2;
		else if (x[j] == '>' && j + 1 < n && x[j + 1] >= '0' && x[j + 1] <= '9') j += 1;
		else continue;
		return x[j] >= '2' && x[j] <= '8' ? x[j] - '0' : 1;
	}
	return 1;
}

int jpegqs_cuda_jpeg_orientation(const uint8_t *data, size_t len, int32_t *orientation) {
	static const char xmp_id[] = "http://ns.adobe.com/xap/1.0/";     /* with its NUL: 29 bytes */
	jq_image im; jq_header h; char err[256]; size_t p = 2, xmp_at = 0, xmp_len = 0, nexif = 0; uint8_t *exif = NULL; int o;
	if (!data || !orientation) { qs_set_host_error("jpegqs_cuda_jpeg_orientation: NULL argument"); return JPEGQS_ERR_ARG; }
	/* the reader's walk up to the first SOS, where Pillow stops too: no entropy-coded byte is read */
	if (jq_read_header(data, len, &im, &h, err)) { qs_set_host_error(err); return JPEGQS_ERR_ARG; }
	jq_free(&im);
	/* the segments before the first SOS, as Pillow's JpegImageFile._open walks them */
	while (p < len) {
		unsigned m; size_t seg;
		if (data[p] != 0xFF) { p++; continue; }
		while (p < len && data[p] == 0xFF) p++;
		if (p >= len) break;
		m = data[p++];
		if (m == 0xDA) break;
		if (m == 0 || m == 0x01 || (m >= 0xD0 && m <= 0xD9)) continue;   /* no length field */
		if (len - p < 2) break;
		seg = (size_t)data[p] << 8 | data[p + 1];
		if (seg < 2 || seg > len - p) break;
		if (m == 0xE1) {
			const uint8_t *s = data + p + 2; size_t sn = seg - 2;
			if (sn >= 6 && !memcmp(s, "Exif\0\0", 6)) {
				/* the first block whole, the later ones without their prefix */
				const uint8_t *add = nexif ? s + 6 : s; size_t an = nexif ? sn - 6 : sn;
				uint8_t *grown = (uint8_t *)realloc(exif, nexif + an + 1);
				if (!grown) { free(exif); qs_set_host_error("jpegqs_cuda_jpeg_orientation: out of memory"); return JPEGQS_ERR_ARG; }
				exif = grown; memcpy(exif + nexif, add, an); nexif += an;
			} else if (sn >= sizeof(xmp_id) && !memcmp(s, xmp_id, sizeof(xmp_id))) {
				xmp_at = p + 2 + sizeof(xmp_id); xmp_len = sn - sizeof(xmp_id);
			}
		}
		p += seg;
	}
	o = exif ? exif_ifd0_orientation(exif, nexif) : EXIF_NO_TAG;
	free(exif);
	if (o == EXIF_RAISES) o = 1;
	else if (o == EXIF_NO_TAG) o = xmp_len ? xmp_orientation(data + xmp_at, xmp_len) : 1;
	*orientation = o;
	return 0;
}
