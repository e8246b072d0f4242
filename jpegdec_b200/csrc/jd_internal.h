/*
 * jd_internal.h -- structures shared between the host C code (jd_host.c, jd_api.c),
 * the device pipeline (jd_device.cu) and the kernels (jd_kernels.cuh).
 */
#ifndef JD_INTERNAL_H
#define JD_INTERNAL_H

#include <stdint.h>
#include "../../include/JPEGDEC.h"
#include "../../include/jpegdec_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define JD_LUT_ENTRIES_H 10496 /* == JD_LUT_ENTRIES in jd_core.h */

/* Host-side result of parsing one JPEG header (all the per-image facts the GPU needs). */
typedef struct {
    int width, height;
    int subsample;          /* 0x00 gray, 0x11, 0x21, 0x12, 0x22 */
    int ncomp;              /* 1 or 3 */
    int mode;               /* 0xC0 baseline, 0xC2 progressive */
    int bpp;
    int restart_interval;   /* MCUs, 0 = none */
    int scan_offset;        /* byte offset of entropy-coded data */
    int orientation, has_thumb, thumb_w, thumb_h, thumb_data, exif;
    int mcu_w, mcu_h;       /* MCU size in pixels */
    int mcus_x, mcus_y;
    int bpm;                /* blocks per MCU */
    int tsel;               /* per comp c: bit 2c = DC table, bit 2c+1 = AC table */
    int tables_ok;          /* scan uses only tables 0/1 (DC and AC) */
    int error;              /* JPEG_* error code when parse fails */
    int approx;             /* first scan's successive-approximation byte (Ah << 4 | Al); progressive files */
    int jfif;               /* a JFIF APP0 segment was seen */
    int adobe;              /* transform byte of the last Adobe APP14 segment, -1 = none */
    JDPARSED p;
} JDInfo;

/* jd_host.c */
int jd_parse_header(const uint8_t *data, int size, int start_offset, JDInfo *info);
/* The same for a batch created with `options`: with JPEGB200_OPT_PROGRESSIVE a progressive file's Huffman tables are not
 * held to the reference's LUT classes (its scans are decoded with jd_prog.h's own tables). */
int jd_parse_header_opt(const uint8_t *data, int size, int start_offset, JDInfo *info, int options);
int jd_check_huffman(const JDInfo *info);                      /* 1 ok, 0 -> JPEG_UNSUPPORTED_FEATURE */
void jd_build_lut(const JDInfo *info, uint16_t *lut /* JD_LUT_ENTRIES_H */);
void jd_build_quant(const JDInfo *info, int16_t *q /* [3][64] natural order, per component */);
uint64_t jd_tables_hash(const JDInfo *info);
uint64_t jd_tables_hash2(const JDInfo *info);
int jd_tables_equal(const JDInfo *x, const JDInfo *y);
const int *jd_aan_table(void);

/* Device-visible per-image descriptor (96 B). */
typedef struct {
    uint32_t scan_off;      /* absolute offset of first entropy byte in the batch buffer */
    uint32_t scan_end;      /* absolute end of this file's bytes */
    uint16_t width, height;
    uint16_t mcus_x, mcus_y;
    uint8_t subsample, ncomp, bpm, tsel;
    uint32_t mcus_per_seg;
    uint32_t nseg;
    uint32_t seg_base;      /* first global segment index */
    uint32_t blk_base;      /* first global block index */
    uint32_t lutset;        /* index of the Huffman LUT set */
    uint32_t out_pitch;     /* bytes */
    uint32_t prog;          /* bit 0: progressive file, only the DC coefficients of its first scan are decoded (reference
                             * JPEGDecodeMCU_P, src/jpeg.inl:1819-2084, 1/8-scale output); bits 8..11: point transform Al */
    uint64_t out_off;       /* byte offset from the output base pointer */
    uint32_t out_w, out_h;  /* output size in pixels after scaling */
    uint32_t status;        /* written by kernels: 0 ok */
    uint32_t err_mcu;
    uint32_t chunk_base;    /* restart-free scans decoded in parallel chunks: first global chunk index ... */
    uint32_t nch;           /* ... and number of chunks (0 = the scan is decoded per restart segment) */
    uint32_t comp_off;      /* offset of this file's first byte in the batch buffer */
    uint32_t nseg_walk;     /* restart intervals the entropy stage walks: nseg, or with a region of interest those that
                             * start at or above the rectangle's last MCU row (jd_roi_plan) */
    uint64_t rec_base;      /* index of this image's first coefficient record: block headers hold record indices relative
                             * to it (jd_core.h JD_REC_INDEX with byte offsets relative to comp_off and image-local slots) */
    /* region of interest (JPEGB200_batchCreateROI); out_w / out_h above are then its size */
    uint16_t roi_x, roi_y;  /* its origin in output pixels (0, 0 without one) */
    uint16_t mcu_x0, mcu_y0;/* first MCU column / row it touches: the IDCT grid starts there */
    uint32_t roi_mcu_end;   /* view descriptors only: 1 + the last MCU (full-image raster index) of the last MCU row it
                             * touches; 0 = no rectangle.  JPEGB200_batchErrMcu does not report a file error at or past this
                             * MCU (jd_view_err_mcu).  File descriptors keep 0: no kernel reads it. */
    uint32_t orient;        /* EXIF transform 1-8 applied by the stores (JPEGB200_batchCreateOriented; 0 / 1 = none).  With
                             * it, roi_x / roi_y and the MCU box are those of the rectangle in the STORED frame, while out_w /
                             * out_h stay the output (upright) size: swapped against the stored rectangle for 5-8. */
} JDImageDesc;

/* What a region of interest (in output pixels: after scaling) means for one image: the MCUs it touches, the restart
 * intervals that must be walked to reach them and the output size.  jd_roi_plan returns 0 for a rectangle that does not
 * lie inside the output image. */
typedef struct {
    int32_t mcu_x0, mcu_y0, mcu_x1, mcu_y1;  /* MCU columns / rows touched, inclusive */
    int32_t nseg_walk;                       /* restart intervals walked (intervals below the last touched row are skipped) */
    int32_t mcu_end;                         /* (mcu_y1 + 1) * MCUs per row */
    int32_t out_w, out_h;                    /* = the rectangle's w, h */
} JDRoiPlan;
int jd_roi_plan(int width, int height, int subsample, int restart_interval, int sshift, const int32_t *rect /* x, y, w, h */,
                JDRoiPlan *plan);
/* EXIF transform k as mirrors of the stored frame followed by an optional transpose (k >= 5): bit k of these masks says
 * whether k mirrors x (stored column sx -> sw - 1 - sx) and y.  2 = mirror x, 3 = both, 4 = y, 5 = transpose, 6 = y then
 * transpose (90 degrees clockwise), 7 = both then transpose, 8 = x then transpose (90 degrees counter-clockwise). */
#define JD_ORIENT_MX 0x18Cu
#define JD_ORIENT_MY 0x0D8u
/* The same for an oriented image.  k: EXIF transform 1-8.  rect: x, y, w, h in the OUTPUT (upright) frame, whose size is the
 * scaled image's with width and height swapped for k = 5-8; NULL = the whole image.  srect receives the rectangle in the
 * stored frame (where the MCUs are), plan is jd_roi_plan's for srect except that out_w / out_h are the output size (w, h).
 * Returns 0 for a k outside 1-8 or a rectangle that does not lie inside the output image. */
int jd_orient_plan(int width, int height, int subsample, int restart_interval, int sshift, int k, const int32_t *rect,
                   int32_t *srect /* x, y, w, h */, JDRoiPlan *plan);

/* The per-image arguments of nv images (or views) of one file, as JPEGB200_batchCreateViews checks them: for view v,
 * ok[v] = 0 when its rectangle does not lie inside the output, its transform ks[v] is outside 1-8 or its resize target
 * out_sizes[2v], [2v+1] is outside 1..65535; plans[v] / srects[4v] are jd_orient_plan's (ks given: the resolved EXIF
 * transforms, 0 = from the file already replaced) or jd_roi_plan's and the rectangle's origin (rois only); rois, ks and
 * out_sizes may each be NULL.  Returns the restart intervals the file's entropy walk covers: the largest nseg_walk of its
 * valid views (all nseg intervals for a view of a batch without rois and orients), 0 if no view is valid. */
int jd_views_plan(int width, int height, int subsample, int restart_interval, int sshift, int nv, const int32_t *rois,
                  const uint8_t *ks, const int32_t *out_sizes, JDRoiPlan *plans, int32_t *srects, int32_t *ok);
/* The first undecodable MCU an image (view) reports, -1 for none.  file_status / file_err_mcu: what jdk_stitch (or
 * jdk_prog_pack) wrote for the view's file, whose walk reaches the deepest of its views; mcu_end: the view's
 * JDRoiPlan.mcu_end (0 = no rectangle).  The view reports the file's error when it has no rectangle or the error lies before
 * mcu_end, as the reference's crop decode, which stops parsing after the rectangle's last MCU row.  A view alone in its file
 * gets the same answer as with several: a view's walked intervals are a prefix of its file's and every MCU before its
 * mcu_end lies in that prefix.  The chunk path's error MCU is judged the same way, wherever its chunk lies. */
int32_t jd_view_err_mcu(uint32_t file_status, uint32_t file_err_mcu, uint32_t mcu_end);
/* How many files, from the first, the next job of JPEGB200_decodeBatchViews takes: always the first, then each next file
 * while the job keeps at most max_views views, at most max_bytes compressed bytes (a negative size counts 0) and, with
 * scratch (per view, may be NULL), at most max_scratch scratch bytes.  views NULL = one view per file.  *nviews receives
 * the job's views; *capped is 1 when the file after the job was left out because of max_views. */
int jd_job_files(int nf, const int32_t *sizes, const int32_t *views, int64_t max_views, int64_t max_bytes,
                 const int64_t *scratch, int64_t max_scratch, int32_t *nviews, int32_t *capped);

/* Resize of one image (JPEGB200_batchCreateResized) from the unresized output S (src_w x src_h) to out_w x out_h: the O(1)
 * facts that size its scratch; the coefficients themselves are computed on the GPU (jd_resize.h, jdk_resize_coeffs).
 * A pass runs only along an axis whose size changes (Pillow skips the other).  The horizontal pass reads source rows
 * ybox0 .. ybox0 + rows - 1 (those the vertical pass's first and last output rows reach) and writes rows x out_w pixels.
 * Pillow 12 runs the vertical pass first for a tall source that shrinks vertically (src_h > 100 src_w, out_h < src_h,
 * both passes needed); the intermediate is then out_h x src_w pixels.  The order changes the rounding, so it is kept. */
typedef struct {
    int32_t need_h, need_v;
    int32_t vfirst;             /* vertical pass first */
    int32_t ksize_h, ksize_v;   /* coefficient table strides (taps of the widest output column / row) */
    int32_t ybox0, rows;        /* source rows of the horizontal pass (all src_h rows when the height does not change) */
    int64_t mid_bytes;          /* intermediate: rows x out_w x bytes per pixel (0 without a horizontal pass) */
    int64_t coef_words;         /* int32 table words: out_w x (ksize_h + 2) and out_h x (ksize_v + 2) for the passes that run */
} JDResizePlan;
/* Returns 0 for a filter other than JPEGB200_RESIZE_* or a size outside 1..65535. */
int jd_resize_plan(int src_w, int src_h, int out_w, int out_h, int filter, int bytes_per_pixel, JDResizePlan *plan);

/* Window of one view (JPEGB200_batchCreateWindow): the crop (x, y, w, h) of R, the resize of S (src_w x src_h) to out_w x
 * out_h, as Pillow's R.crop((x, y, x + w, y + h)).  Window columns x0 .. x1 - 1 and rows y0 .. y1 - 1 lie inside R; the
 * others are fill (all four 0 when the window reads no pixel of R).  The support (sx, sy, sw, sh) is the rectangle of S the
 * in-image outputs read: along a resampled axis from the first one's xmin to the last one's xmin + taps (jd_rs_bounds with
 * the full sizes), along an axis Pillow does not resample the window's in-image span; 1 x 1 at S's origin when the window
 * reads nothing.  rp holds the passes: need_h, need_v, vfirst and the strides on the full sizes (Pillow decides there, and
 * the order changes the rounding), ybox0 = 0 and rows = sh (every support row), and the intermediate and coefficient tables
 * for the window only. */
typedef struct {
    int32_t sx, sy, sw, sh;
    int32_t x0, x1, y0, y1;
    JDResizePlan rp;
} JDWindowPlan;
/* Returns 0 for what jd_resize_plan refuses and for a window side outside 1..65535. */
int jd_window_plan(int src_w, int src_h, int out_w, int out_h, int filter, const int32_t *window, int bytes_per_pixel,
                   JDWindowPlan *plan);

/* Box resize of one view (JPEGB200_batchCreateBox): Pillow's resize(out, filter, box, reducing_gap) of S (sw x sh) as its
 * Python code decides it, in double: factor = int(box extent / out / gap) or 1 per axis; with a factor above 1 the region
 * _get_safe_box(out, filter, box) of S is reduced (jd_reduce.h) and the box carried into the reduced frame; then the C
 * resize of the resize source (the reduced image, or S) with that box as float, vertical pass first for a source more
 * than 100 times taller than wide that shrinks vertically (two calls in Pillow, the same passes here). */
typedef struct {
    int32_t fx, fy;             /* reduce factors; 1 x 1 = no reduce */
    int32_t rx0, ry0, rx1, ry1; /* the reduced region of S (the safe box), S itself without a reduce */
    int32_t rw, rh;             /* the resize source: ceil(region / factor) */
    float box[4];               /* x0, y0, x1, y1 of the resize in the source's frame, as Pillow's C resize receives it */
    JDResizePlan rp;            /* the passes from the source to out_w x out_h: need_h / need_v are true for any box that
                                 * does not start at 0 and end at the output size (Pillow's C test) */
} JDBoxPlan;
/* box: x0, y0, x1, y1 in S; gap: reducing_gap, 0 = None.  Returns 0 for what Pillow refuses with a ValueError (a box
 * value that is not finite, a float box with a negative offset, past sw / sh or with a negative extent, gap < 1), for a
 * reduce to an empty image or of boxes of 2^23 pixels or more, and for jd_resize_plan's refusals.  The box is checked in
 * S's frame: one past the edge is refused even where Pillow's reduce would carry it inside the reduced image. */
int jd_box_plan(int sw, int sh, int out_w, int out_h, int filter, const double *box, double gap, int bytes_per_pixel, JDBoxPlan *plan);
/* The window of a boxed view: box->rp's passes, the whole resize source as the support (no narrowing), the intermediate and
 * tables for the window.  0 for a window side outside 1..65535. */
int jd_window_box(const JDBoxPlan *box, int out_w, int out_h, const int32_t *window, int bytes_per_pixel, JDWindowPlan *plan);
/* Batch-level rule of JPEGB200_batchCreateBox: boxes or reducing_gaps need out_sizes.  0 with a message otherwise. */
int jd_check_box(const int32_t *out_sizes, const double *boxes, const double *gaps, char *msg, int msg_len);

/* Colour operations of one view (JPEGB200_batchCreateColor, jd_color.h): row = its JPEGB200_COLOR_MAX_OPS entries.  Writes
 * the plan the kernels run -- factors as float bits, hue shift bytes, solarize thresholds as the count of bytes below them,
 * the segments cut at each contrast and each blur; on a gray view (gray != 0) saturation, hue and grayscale are dropped.
 * Blurs of radius 0 are dropped, negative radii planned as |r|, and each blur's constants written to blur (when not NULL)
 * at its op slot.  Returns 0 for an unknown op, an argument that is not finite, a hue outside [-0.5, 0.5], or a blur
 * radius whose float32 magnitude is 2^31 or more.  jd_color_plan is the same without the blur constants.
 * jd_color_plan_aug also plans the auto-augment operations (jd_augment.h) of a w x h view: the list is cut before each
 * sharpness, autocontrast, equalize and geometric op; posterize is planned as its mask; each geometric op's 16.16 mapping
 * goes to aug (when not NULL) at its op slot.  It also returns 0 for a posterize argument that is not an integer in 0 .. 8,
 * and, when aug is not NULL, for a geometric op on a view with a side above JD_AU_MAX_SIDE or whose mapping does not fit
 * 32 bits.  jd_color_plan_blur is jd_color_plan_aug with aug NULL.
 * Every variant plans the JPEG ops (JPEGB200_COLOR_JPEG, _444, _422; jd_jpegop.h) as a cut with arg q, and returns 0 for a
 * q that is not an integer in 1 .. 100.
 * jd_color_plan_rs also plans the geometric ops flagged JPEGB200_COLOR_BILINEAR or _BICUBIC: cut like the NEAREST ones,
 * each one's matrix (jd_aug_matrix) into rs at its op slot.  It returns 0 for a flag that is not exactly one of the two on
 * a geometric code, and for a flagged op on a view with a side above JD_AU_MAX_SIDE.  jd_color_plan_aug is
 * jd_color_plan_rs with rs NULL, which refuses every flagged op, as the plans without rs always have.
 * jd_color_plan_warp also plans JPEGB200_COLOR_AFFINE / _PERSPECTIVE (bare or with one filter flag), whose arguments are
 * warp[k] for op slot k of the row: cut like the geometric ops, the coefficients and the clamped fill into wp, and a
 * NEAREST affine with b or d non-zero as its 16.16 mapping into aug, at the op's plan slot.  It returns 0 for both filter
 * flags together, a non-finite coefficient, a view side above JD_AU_MAX_SIDE and such an affine where Pillow does not
 * take its 16.16 form (|x a + y b + c| or |x d + y e + f| at least 32768 at a corner (0 or w, 0 or h) of the view).  jd_color_plan_rs is jd_color_plan_warp with warp and wp NULL, which refuses both codes. */
#include "jd_color.h"
#include "jd_augment.h"
int jd_color_plan_warp(const JPEGB200_ColorOp *row, const JPEGB200_WarpArgs *warp, int gray, uint32_t w, uint32_t h,
                       JDColorPlan *plan, JDBlurPlan *blur, JDAugPlan *aug, JDResamplePlan *rs, JDWarpPlan *wp);
/* jd_au_walk_table, built here without FMA contraction: the table jdk_warp reads for a NEAREST affine with b = d = 0 */
void jd_walk_table(const double *c, uint32_t w, uint32_t h, int16_t *tab);
int jd_color_plan_rs(const JPEGB200_ColorOp *row, int gray, uint32_t w, uint32_t h, JDColorPlan *plan, JDBlurPlan *blur,
                     JDAugPlan *aug, JDResamplePlan *rs);
int jd_color_plan_aug(const JPEGB200_ColorOp *row, int gray, uint32_t w, uint32_t h, JDColorPlan *plan, JDBlurPlan *blur,
                      JDAugPlan *aug);
int jd_color_plan_blur(const JPEGB200_ColorOp *row, int gray, JDColorPlan *plan, JDBlurPlan *blur);
int jd_color_plan(const JPEGB200_ColorOp *row, int gray, JDColorPlan *plan);
/* the inverse matrix Pillow's transform gets for geometric op `op` with magnitude m on a w x h image (torchvision's
 * _apply_op: _get_inverse_affine_matrix, or Image.rotate's matrix) */
void jd_aug_matrix(int op, double m, uint32_t w, uint32_t h, double *mat);
/* Python's round(x, 15) */
double jd_round15(double x);
/* GaussianBlur(r)'s box half-width and 24-bit weights for r = |radius| as float32, 0 < r < 2^31 (0 past that) */
int jd_blur_consts(float r, JDBlur *out);
/* Batch-level rule of JPEGB200_batchCreateColor: no operation on RGB565, dithered pixel types or padded output (checked
 * over the nv rows).  0 with a message otherwise. */
int jd_check_color(int pixel_type, int options, int64_t nv, const JPEGB200_ColorOp *color_ops, char *msg, int msg_len);

/* Coefficient records an image's entropy walks can address above its record base: the largest JD_REC_INDEX + JD_REC_CAP
 * (jd_core.h) over its restart segments (slots 0 .. nseg - 1, each ending at or before the file's end) and the chunks of a
 * restart-free scan (slots nseg .. nseg + nch - 1, 512 bytes each from scan_offset), computed in 64 bits.  Those indices
 * are 32-bit: JPEGB200_batchCreate refuses an image whose extent passes 2^32, whose last slots would otherwise overwrite
 * the records of its first ones.  Files under 512 MiB reach it only through the 128 spare records per restart interval.
 * (jd_device.cu; declared here so that the CPU tests can call it.) */
uint64_t jd_rec_extent(uint64_t size, uint32_t scan_offset, uint32_t nseg, uint32_t nch);

/* ---- progressive files decoded from all their scans (JPEGB200_OPT_PROGRESSIVE, jd_prog.h, DESIGN.md 4.3.1) ---- */
#define JD_PROG_MAX_SCANS 64
#define JD_PROG_MAX_TABS (3 * JD_PROG_MAX_SCANS)
#define JD_PROG_MAX_BLOCKS (1u << 26)   /* plane indices (block * 64 + k) stay 32-bit */
/* Canonical Huffman decoder of one table as a scan uses it: any valid code of 1-16 bits. */
typedef struct {
    uint16_t look[256];     /* next 8 bits -> code length << 8 | symbol; 0 = a longer code (or no code) */
    int32_t maxcode[17];    /* [l]: largest code of length l, -1 = none */
    int32_t valoff[17];     /* [l]: the symbol of code c of length l is val[c + valoff[l]] */
    uint8_t val[256];
} JDProgHuff;
/* One scan of a progressive file.  Blocks of the plane are numbered like the baseline walk's block headers: MCU by MCU,
 * luma blocks in raster order inside the MCU, then Cb, Cr. */
typedef struct {
    uint32_t start, end;    /* entropy bytes [start, end) up to the next marker that is not RSTn: file offsets from
                             * jd_prog_parse, batch-buffer offsets on the device */
    uint32_t img;           /* file index in the batch */
    uint32_t row_limit;     /* the walk stops before this MCU row (regions of interest and views) */
    uint16_t width, height, mcus_x, mcus_y;
    uint16_t restart;       /* restart interval of this scan (MCUs, or blocks of a one-component scan), 0 = none */
    uint8_t subsample, ncomp, bpm;
    uint8_t ncs, ss, se, ah, al, wave;
    uint8_t comp[3];        /* frame component index of each scan component */
    uint32_t tab[3];        /* decoder of each scan component (DC or AC table): index into the table list */
} JDProgScan;
/* Scan list of a progressive file whose header jd_parse_header_opt accepted (start: where that parse started).  Fills
 * scans (JD_PROG_MAX_SCANS) and tabs (JD_PROG_MAX_TABS, *ntabs used; scans[].tab index them), gives each scan its wave
 * (a scan comes after every earlier scan of one of its components whose coefficient range overlaps its own) and returns
 * the number of scans, or minus a JPEG_* status: JPEG_DECODE_ERROR for a file that breaks the progression rules of T.81
 * G.1.1.1, JPEG_UNSUPPORTED_FEATURE for more than JD_PROG_MAX_SCANS scans, more than JD_PROG_MAX_BLOCKS blocks or a
 * chroma sampling other than 1x1. */
int jd_prog_parse(const uint8_t *data, int size, int start, const JDInfo *info, JDProgScan *scans, JDProgHuff *tabs, int *ntabs);
/* Coefficient records a progressive image may need (the pack refuses more): every stored coefficient costs at least two
 * bits of some scan (a code and a magnitude or sign bit) and at most two records, so 8 per entropy byte, plus the 126 that
 * the one block where a failing scan stops may hold without paying for them (zero bits past its data), per scan; at most
 * 2^32 - 1 (block headers hold 32-bit record indices). */
uint64_t jd_prog_rec_cap(uint64_t entropy_bytes, uint32_t nscans);

/* ---- libjpeg's default decompression (JPEGB200_OPT_LIBJPEG, jd_ljpeg.h, DESIGN.md 4.2.6) ---- */
/* 1 when libjpeg would convert the file's 3 components from YCbCr (jdapimin.c's inference: a JFIF APP0 means YCbCr; else
 * an Adobe APP14 decides, transform 0 = RGB; else component ids 'R', 'G', 'B' mean RGB and anything else YCbCr), 0 when
 * they are R, G, B already.  Gray files: 1. */
int jd_lj_is_ycc(const JDInfo *info);
/* The raw DQT values of each component's own table, column-major per component ([c * 64 + col * 8 + row]), the layout of
 * the batch's quant array. */
void jd_lj_quant(const JDInfo *info, int32_t *q /* [3][64] */);
/* Extends a view's plan (jd_roi_plan / jd_orient_plan for srect: x, y, w, h in the stored frame at full scale) to the MCUs
 * a libjpeg decode of the rectangle reads: fancy upsampling reads, in each subsampled direction, the neighbouring chroma
 * sample of the rectangle's first and last pixel (the one before an even first pixel, the one after an odd last pixel,
 * clamped to the component's real samples; none in the narrow fallback), which may lie in the next MCU.  For vertically
 * subsampled files the walk and mcu_end then reach the last MCU row read. */
void jd_lj_plan_extend(int width, int height, int subsample, int restart_interval, const int32_t *srect, JDRoiPlan *plan);
/* The same for a view decoded at 1 / 2^shift (JPEGB200_batchCreateDraft): srect in the stored frame of the scaled image, plan
 * jd_roi_plan's at that shift.  Upsampling reads a neighbouring chroma sample only along an axis that is still upsampled at
 * this scale with the fancy filter (jd_ljpeg.h); shift 0 is jd_lj_plan_extend. */
void jd_lj_plan_extend_s(int width, int height, int subsample, int restart_interval, int shift, const int32_t *srect,
                         JDRoiPlan *plan);
/* Per-view scale denominators of JPEGB200_batchCreateDraft: 1 with draft == NULL or with JPEGB200_OPT_LIBJPEG; 0 with a
 * message for a draft without JPEGB200_OPT_LIBJPEG.  A value other than 1, 2, 4 or 8 is not refused here: that view alone
 * gets JPEG_INVALID_PARAMETER (jd_draft_shift). */
int jd_check_draft(int options, const uint8_t *draft, char *msg, int msg_len);
/* log2 of a draft denominator (1, 2, 4, 8 -> 0..3), -1 for any other value */
static inline int jd_draft_shift(uint8_t s) { return s == 1 ? 0 : s == 2 ? 1 : s == 4 ? 2 : s == 8 ? 3 : -1; }
/* Per image of a libjpeg batch: its MCU box and where its planes live in the batch's plane scratch (jd_ljpeg.h). */
typedef struct {
    uint64_t plane_off;     /* byte offset of the box's planes (256-byte aligned) */
    uint32_t mx0, my0;      /* the box's first MCU column / row */
    uint32_t nmx, nmy;      /* its size in MCUs; 0 = nothing to decode (a failed image) */
    uint32_t ycc;           /* jd_lj_is_ycc */
    uint32_t shift;         /* the view's scale 1 / 2^shift (JPEGB200_batchCreateDraft); 0 = full scale */
} JDLjDesc;

/* A caller's destination for image `index` (only named in the message): row_bytes is the tight pitch
 * (JPEGB200_batchOutputBytes), pitch <= 0 means tight.  device != 0: `out` is written by the kernels.  Returns 1, or 0 with
 * a message in msg[msg_len] (see JPEGB200_batchSetOutput / JPEGB200_decodeBatch for the rules). */
int jd_check_output(int index, int pixel_type, int64_t row_bytes, const void *out, int64_t pitch, int device,
                    char *msg, int msg_len);

#define JPEGB200_OPT_PADDED 0x10000 /* internal option bit (the single-image API, jd_api.c): write the whole MCU-aligned frame */

/* JPEG_LUMA_ONLY turns the colour pixel types into 8-bit gray (jpeg.inl:4991) */
static inline int jd_fold_luma_only(int pixel_type, int options)
{
    return ((options & JPEG_LUMA_ONLY) && pixel_type < EIGHT_BIT_GRAYSCALE) ? EIGHT_BIT_GRAYSCALE : pixel_type;
}
/* The images of a batch or call of nfiles files: the sum of views[f] (each at least 1, at most INT32_MAX in all; `per` names
 * "batch" or "call" in that message), nfiles without views.  -1 with a message. */
int64_t jd_count_views(int nfiles, const int32_t *views, const char *per, char *msg, int msg_len);
/* Which combinations of pixel type, options and features (views, a tensor spec, out_sizes with `filter`, rois, orients) a
 * batch accepts: JPEGB200_batchCreateViews' argument rules.  Returns 1 and the batch's image count in *nviews, or 0 with the
 * message of the first rule broken: an invalid parameter, JPEGB200_OPT_LIBJPEG's own rules, the view counts, then
 * per feature what it is not supported with (views, tensor and its spec, resize and its filter, rois / orients with
 * dithered types, rois / orients with padded output). */
int jd_check_batch_features(int pixel_type, int options, int nfiles, const int32_t *views, int has_rois, int has_orients,
                            int has_out_sizes, int filter, const JPEGB200_TensorSpec *spec, int64_t *nviews, char *msg,
                            int msg_len);

/* Tensor output (JPEGB200_batchCreateTensor).  The byte order of an RGB8888 output: 1 = B,G,R,A, 0 = R,G,B,A.  The
 * SSE2-build arithmetic stores B,G,R,A at full scale for 3-component 4:2:0 and 4:4:4 files (its SIMD colour paths);
 * every other case takes the scalar colour code, which stores R,G,B,A.  Depends on the image, so it is asked per image. */
int jd_rgb8888_is_bgr(int arith, int sshift, int ncomp, int subsample);
/* Element size of a JPEGB200_DT_* (0 = unknown). */
int jd_tensor_elt(int dtype);
/* 1 if spec is usable with `channels` output channels (1 or 3), else 0 with a message. */
int jd_tensor_check(const JPEGB200_TensorSpec *spec, int channels, char *msg, int msg_len);
/* The 3 x 256 output elements (channel-major, jd_tensor_elt(spec->dtype) bytes each, little-endian bit patterns) of byte
 * value x in output channel c, in plain IEEE float32 arithmetic (JPEGB200_batchCreateTensor's formula).  The kernel only
 * looks these up.  Returns the element size, 0 for an unknown dtype or scale. */
int jd_tensor_table(const JPEGB200_TensorSpec *spec, void *out);
/* A caller's tensor destination (device memory): see JPEGB200_batchSetOutputTensor.  row_bytes: the tight row, rows: H,
 * chw: planar layout.  Returns 1, or 0 with a message. */
int jd_check_tensor_output(int index, int elt, int64_t row_bytes, int64_t rows, int chw, const void *out, int64_t pitch,
                           int64_t plane_stride, char *msg, int msg_len);

#ifdef __cplusplus
}
#endif
#endif
