/*
 * jpegcoef.h - a small JPEG coefficient codec (ITU-T T.81 Huffman modes, 8-bit samples).
 *
 * The reference CLI gets its coefficient arrays from libjpeg (jpeg_read_coefficients /
 * jpeg_write_coefficients, reference quantsmooth.c:548-596).  libjpeg's headers are not
 * available in this build image, so the `jpegqs` tool here carries its own front/back end
 * (SURVEY.md 8f row f1): it parses baseline, extended-sequential and progressive Huffman
 * JPEGs into exactly the structures do_quantsmooth consumes (a jpeg_decompress_struct
 * with an in-memory jpeg_memory_mgr and one virtual block array per component) and writes the
 * arrays back as a sequential Huffman JPEG with libjpeg's own JFIF / Adobe header markers
 * (jcmarker.c write_file_header) followed by the copied APPn/COM markers.  No pixels are decoded.
 * Arithmetic-coded, lossless, hierarchical and 12-bit files are rejected.
 */
#ifndef JPEGCOEF_H
#define JPEGCOEF_H

#include <stddef.h>
#include <jpeglib.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct jq_marker {
	int code;                    /* 0xE0..0xEF (APPn) or 0xFE (COM) */
	size_t len;                  /* payload bytes (without the 2 length bytes) */
	unsigned char *data;
	struct jq_marker *next;
} jq_marker;

typedef struct jq_image {
	struct jpeg_decompress_struct cinfo;     /* what do_quantsmooth reads and rewrites */
	jvirt_barray_ptr coef_arrays[MAX_COMPONENTS];
	jq_marker *markers;                      /* in file order */
	int progressive;                         /* the input was SOF2 */
	int restart_interval;                    /* of the input (not reproduced on output) */
	int comp_id[MAX_COMPONENTS];             /* component identifiers of the frame header */
	/* what libjpeg keeps in saw_JFIF_marker / JFIF_*_version / density / saw_Adobe_marker /
	 * Adobe_transform (jdmarker.c) and jpeg_copy_critical_parameters hands to the writer */
	int saw_jfif, jfif_major, jfif_minor, density_unit, x_density, y_density;
	int saw_adobe, adobe_transform;
	int warnings;                            /* recoverable anomalies (libjpeg: err->num_warnings) */
	void *priv;
} jq_image;

/* copy: 0 = no markers, 1 = COM only, 2 = COM + APPn (reference quantsmooth.c:541-546).
 * Returns 0, or -1 with a message in err (>= 256 bytes). */
int jq_read(const unsigned char *data, size_t len, int copy, jq_image *im, char *err);

/* Encodes im->cinfo + arrays (normally im->coef_arrays, or the arrays do_quantsmooth left in
 * its coef_arrays argument) as one sequential Huffman JPEG.  optimize != 0 builds optimal
 * Huffman tables (the CLI's -o, reference quantsmooth.c:553).  *out is malloc'd. */
int jq_write(jq_image *im, jvirt_barray_ptr *arrays, int optimize, unsigned char **out, size_t *outlen, char *err);

void jq_free(jq_image *im);

/* What is in force at the first SOS: its component order and table selectors, the Huffman
 * tables as DHT sent them (bits[0] unused), the restart interval and where the entropy-coded
 * data starts. */
typedef struct {
	int sof;                             /* 0xC0, 0xC1 or 0xC2 */
	int ncomp, ci[4], td[4], ta[4];      /* scan components (frame indices) and selectors */
	int dc_present[4], ac_present[4];
	unsigned char dc_bits[4][17], dc_val[4][256], ac_bits[4][17], ac_val[4][256];
	int restart_interval;
	size_t entropy_offset;
} jq_header;

/* jq_read's marker walk up to the first SOS: fills im->cinfo (frame, quant tables, colour space)
 * and hdr without reading entropy-coded data and without allocating coefficient arrays.  Returns 0,
 * or -1 with a message in err.  im must be released with jq_free. */
int jq_read_header(const unsigned char *data, size_t len, jq_image *im, jq_header *hdr, char *err);

/* jq_read's marker walk over the whole file without decoding any entropy-coded data (each scan is
 * skipped to the next marker): fills im->cinfo, the colour space, the JFIF / Adobe fields and the
 * markers copied at level `copy`, as jq_read does, but allocates no coefficient arrays.  Returns 0
 * or -1 with a message in err.  im must be released with jq_free. */
int jq_read_markers(const unsigned char *data, size_t len, int copy, jq_image *im, char *err);

/* One scan as jq_read_scans records it: what jq_read's decoder would be handed at its SOS (the
 * tables and restart interval in force), and its entropy-coded bytes [offset, end), end the next
 * marker that is not RSTn (the file's end when none follows). */
typedef struct {
	int sof;                             /* the frame's SOF code: 0xC0, 0xC1 or 0xC2 */
	int ncomp, ci[4], td[4], ta[4], Ss, Se, Ah, Al;
	int dc_present[4], ac_present[4];
	unsigned char dc_bits[4][17], dc_val[4][256], ac_bits[4][17], ac_val[4][256];
	int restart_interval;
	size_t offset, end;
} jq_scanrec;

/* jq_read_markers that also records the scans: recs[0 .. cap), *nrec = all scans found (may exceed
 * cap).  Returns 0 or -1 with a message in err.  im must be released with jq_free. */
int jq_read_scans(const unsigned char *data, size_t len, int copy, jq_image *im, jq_scanrec *recs, int cap, int *nrec, char *err);

/* The bytes jq_write puts before its first DQT: SOI, the JFIF APP0 or Adobe APP14 of the colour
 * space, the copied markers.  *out is malloc'd.  Returns 0 or -1 (out of memory). */
int jq_prefix(const jq_image *im, unsigned char **out, size_t *outlen);

/* worker threads of the codec: 0 = one per processor (at most 16).  The writer codes segments of
 * MCU rows on them; the reader decodes sequential (SOF0/SOF1) scans on them - restart intervals as
 * they are, scans without restart markers by speculative parsing of chunks that are stitched where
 * they synchronize (jpegcoef.c) - from four threads up, and the scans of a progressive file side by
 * side where they touch different coefficients.  Neither the coefficients read nor the
 * bytes written depend on the number.  The environment variable JPEGQS_CODEC_THREADS overrides;
 * JPEGQS_SERIAL_DECODE=1 keeps the reader on one thread, JPEGQS_CODEC_TRACE=1 reports the path taken. */
void jq_set_threads(int n);

#ifdef __cplusplus
}
#endif
#endif
