/*
 * jpegdec_b200.h -- batch / device-resident extension of the JPEGDEC C API and the
 * thin host->CUDA FFI underneath it.  Plain C ABI: pointers and sizes only.
 *
 * Why it exists: the reference's hot path -- DecodeJPEG (src/jpeg.inl:4946-5357)
 * driving JPEGDecodeMCU (:2090-2274), JPEGIDCT (:2278-2798), JPEGPutMCU* (:2799-4868)
 * and JPEGDither (:4871-4940) -- decodes one image per call on one core.  An H100 needs
 * ~10^5 independent restart segments in flight, so the throughput path takes a *batch*
 * of images per call.  JPEG_decode() (include/JPEGDEC.h) is this API with n = 1 plus
 * the reference's callback / framebuffer semantics replayed on the host.
 *
 * Per stage, which reference function it replaces:
 *   jdk_prescan        <- JPEGFilter marker handling (:1431-1540) + restart bookkeeping (:5337-5348)
 *   jdk_entropy        <- JPEGDecodeMCU (:2090-2274) incl. the 64-bit window behaviour; for progressive files the DC part
 *                         of JPEGDecodeMCU_P (:1819-1884); parse-only / low-frequency-only variants for 1/8 and 1/4 scale
 *   jdk_stitch/_patch  <- cross-segment window phase of the same function (SURVEY.md A.2)
 *   jdk_unstuff, jdk_chunk_* <- the same for scans without restart markers (chunk-parallel, self-synchronising)
 *   jdk_idct_tb, jdk_idct_color <- JPEGIDCT + DC-only shortcut (:5146-5154) + JPEGPutMCU22/11/12/21/Gray/8BitGray
 *   jdk_scaled         <- the 1/4 and 1/8 paths of the above (:2305-2326, :3323-3396, :3627-3748)
 *   jdk_dither         <- JPEGDither (:4871-4940)
 *   jdk_resize_*, jdk_tensor <- no reference counterpart: Pillow's resize and torchvision's to_tensor / Normalize
 */
#ifndef JPEGDEC_B200_H
#define JPEGDEC_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct JPEGB200_CTX JPEGB200_CTX;     /* one per (process, GPU) */
typedef struct JPEGB200_BATCH JPEGB200_BATCH; /* one decode job: n images, one pixel type / option set */

/* batch flags */
#define JPEGB200_OUT_DEVICE 1   /* output pointers are device pointers (pixels stay in HBM) */

/* Option bit (with the JPEG_* options of JPEGDEC.h; every batch entry point and JPEG_decode take it): decode progressive
 * (SOF2) files from all of their scans, at every scale, pixel type, rectangle, orientation, resize, tensor spec and view
 * count.  Image i's output is then what the baseline file B with the same quantised coefficients, quant tables, geometry
 * and EXIF data decodes to, with B's coefficients exact (no bit-window truncation: a progressive decoder has none) and
 * the IDCT shortcuts taken from the final coefficients' nonzero positions; at 1/8 scale the DC is the fully refined one.
 * An AC magnitude of 2048 or more after all refinements is a decode error at its block (the baseline rule).  Baseline
 * files decode byte for byte as without the bit.  Status: a file that breaks the progression rules (T.81 G.1.1.1) gets
 * JPEG_DECODE_ERROR; more than 64 scans or more than 2^26 blocks JPEG_UNSUPPORTED_FEATURE; a file whose coefficient plane
 * (128 bytes per block of device memory) cannot be allocated JPEG_ERROR_MEMORY, and the batch goes on.  A block is
 * undecodable when it is corrupt or needs bits past its scan's data; with R the lowest MCU row holding a first
 * undecodable block of any scan, the image gets JPEG_DECODE_ERROR with JPEGB200_batchErrMcu = R x MCUs per row (the
 * region-of-interest and view rules below apply to that MCU), and every MCU row above R decodes exactly.  Work: one
 * GPU thread per (file, scan) in waves (jdk_prog_scan, timed as JPEGB200_T_ENTROPY and counted in JPEGB200_C_SEGMENTS),
 * then jdk_prog_pack writes the baseline walk's block headers and records (JPEGB200_T_STITCH, JPEGB200_C_RECORD_BYTES);
 * progressive images add nothing to JPEGB200_C_EVENTS.  Dithered types: the error diffusion starts, as for every file,
 * from the file's own DHT bytes (a reference quirk); they are those of the progressive file, not of B, so the dithered
 * output equals B's only when B carries the same tables.  Without the bit a progressive file gives the reference's 1/8 DC
 * thumbnail of its first scan, or JPEG_UNSUPPORTED_FEATURE at other scales. */
#define JPEGB200_OPT_PROGRESSIVE 0x100
/* options bit of every batch entry point (JPEGB200_batchCreate* / JPEGB200_decodeBatch*, views included): image i's output
 * is libjpeg-turbo's default decompression of the file -- what PIL.Image.open(f).convert("RGB") and
 * torchvision.io.decode_jpeg on the CPU return -- instead of the reference's pixels:
 *   - IDCT: jpeg_idct_islow on coefficients dequantized with the raw DQT values of each component's own table.  The
 *     coefficients are exact: the reference's bit-window truncation is not applied (JPEGB200_C_EVENTS is 0;
 *     JPEGB200_C_EVENT_CANDIDATES still counts the candidate reads the walk met).  Equal to x86-64 libjpeg-turbo's SIMD islow on every block whose dequantized coefficients
 *     and first-pass outputs fit in 16 bits and whose results lie in [-256, 511] before the +128: every block an encoder
 *     writes from 8-bit samples.  Outside it, jidctint.c's 32-bit arithmetic clamped to 0..255.
 *   - Upsampling: libjpeg's fancy triangle filters (h2v2, h2v1, h1v2), edges replicating the component's last real
 *     sample; plain replication for h2v1 / h2v2 components at most 2 samples wide, as libjpeg does.
 *   - Colour: jdcolor.c's YCbCr -> RGB tables, clamped.  Colour space as libjpeg infers it: a JFIF APP0 means YCbCr;
 *     else an Adobe APP14 decides (transform 0: RGB, no conversion); else component ids 'R','G','B' mean RGB and any
 *     other ids YCbCr.
 *   - Pixel types: RGB8888 stores R, G, B, 0xFF for every file (a gray file: Y, Y, Y, 0xFF = convert("RGB")), so tensors
 *     get R, G, B without a swap; EIGHT_BIT_GRAYSCALE stores Y (= decode_jpeg(mode=GRAY)).  An RGB-space file decoded to
 *     EIGHT_BIT_GRAYSCALE gets JPEG_UNSUPPORTED_FEATURE.
 *   - Composes with rectangles, orientations, resize, tensors, views and JPEGB200_OPT_PROGRESSIVE (whose coefficients are
 *     exact too), all of which work on this image instead of the reference's.
 *   - Rectangles: the rectangle equals the same rectangle of the full decode under the bit.  Fancy upsampling reads, in
 *     each subsampled direction, the chroma sample next to the rectangle's first and last pixel, which may lie in the
 *     neighbouring MCU: those MCUs are transformed too, and the status reports an error iff the full decode's first
 *     undecodable MCU lies in an MCU row at or above the last MCU row the rectangle reads (its own last row, or the one
 *     below it).  Restart intervals below that row are not walked.
 *   - Refused (NULL with a message): RGB565 and dithered pixel types, JPEG_SCALE_* (libjpeg's scaled IDCTs are other
 *     algorithms), JPEG_EXIF_THUMBNAIL and JPEG_LUMA_ONLY.
 *   - Work: jdk_lj_idct writes 8-bit planes of each image's MCU box into device scratch (MCUs x blocks x 64 bytes), then
 *     jdk_lj_color upsamples, converts and stores; both are timed as JPEGB200_T_IDCT.  JPEGB200_decodeBatch counts the
 *     planes in its per-job scratch bound. */
#define JPEGB200_OPT_LIBJPEG 0x200

/* stage indices for JPEGB200_batchGetTimings (milliseconds, CUDA events on the batch stream) */
enum {
    JPEGB200_T_H2D = 0,
    JPEGB200_T_PRESCAN,
    JPEGB200_T_ENTROPY,
    JPEGB200_T_STITCH,
    JPEGB200_T_IDCT,
    JPEGB200_T_DITHER,         /* the pixel passes after the IDCT: dither, or resize and tensor conversion (dither never
                                  occurs with either) */
    JPEGB200_T_D2H,
    JPEGB200_T_TOTAL,
    JPEGB200_NUM_TIMINGS
};

/* counters for JPEGB200_batchGetCounters */
enum {
    JPEGB200_C_LAUNCHES = 0,   /* kernels launched by the last batchDecode */
    JPEGB200_C_SEGMENTS,
    JPEGB200_C_BLOCKS,
    JPEGB200_C_EVENTS,         /* coefficients rewritten because the reference reads them through a truncated bit window */
    JPEGB200_C_COMPRESSED_BYTES,
    JPEGB200_C_OUTPUT_BYTES,
    JPEGB200_C_RECORD_BYTES,   /* coefficient-record bytes written by the entropy kernel (restart-segment path) */
    JPEGB200_C_H2D_BYTES,
    JPEGB200_C_D2H_BYTES,
    JPEGB200_C_EVENT_CANDIDATES, /* reads that are truncated for at least one possible window phase (examined, not all applied) */
    JPEGB200_NUM_COUNTERS
};

/* ---- context ---- */
JPEGB200_CTX *JPEGB200_create(int device, int arith_mode);
void JPEGB200_destroy(JPEGB200_CTX *ctx);
const char *JPEGB200_lastErrorString(JPEGB200_CTX *ctx);
int JPEGB200_deviceCount(void);
void *JPEGB200_hostAlloc(size_t bytes);   /* pinned host memory for inputs/outputs */
void JPEGB200_hostFree(void *p);
/* Host placement on multi-socket boxes (optional, never needed for correctness).  numaNode: the host NUMA node the
 * context's GPU hangs off (-1 unknown).  bindHostToDevice: pins the CALLING thread to that node's CPUs (within the CPUs the
 * process may use) and prefers the node for its allocations, so that pinned buffers allocated afterwards and the thread
 * that drives the copies sit next to the GPU; returns the number of CPUs in the new mask, 0 = nothing changed.
 * The reference has no counterpart: its decoder runs where the caller's thread runs (src/JPEGDEC.cpp:157-224). */
int JPEGB200_numaNode(JPEGB200_CTX *ctx);
int JPEGB200_bindHostToDevice(JPEGB200_CTX *ctx);
/* device memory for JPEGB200_OUT_DEVICE outputs (plain cudaMalloc / cudaFree / synchronous cudaMemcpy on the context's GPU) */
void *JPEGB200_deviceAlloc(JPEGB200_CTX *ctx, size_t bytes);
void JPEGB200_deviceFree(JPEGB200_CTX *ctx, void *p);
int JPEGB200_deviceRead(JPEGB200_CTX *ctx, void *host_dst, const void *dev_src, size_t bytes);
/* 64-bit digests of n device byte ranges (starts 8-byte aligned), computed on the GPU: digest = sum over the 8-byte
 * little-endian words w[i] (tail zero padded) of mix64(w[i] ^ i * 0x9E3779B97F4A7C15) mod 2^64, mix64 = splitmix64's
 * finaliser.  Lets a caller check device-resident pixels against digests of reference output without a D2H of the pixels. */
int JPEGB200_digestDevice(JPEGB200_CTX *ctx, const void *const *dev_ptrs, const int64_t *lengths, int n, uint64_t *digests);

/* ---- batch job ---- */
/* Parses the n headers on the host (no GPU work).  datas[i]/sizes[i]: JPEG files in host memory
 * (pinned memory makes the upload a straight DMA; files that sit back to back are uploaded with one copy).
 * pixel_type / options as in JPEGDEC.h.  At most 3 GiB of compressed bytes per batchCreate (JPEGB200_decodeBatch
 * takes any amount and splits it); a single file may be at most 512 MiB.  Within those byte limits a batch may hold
 * any number of images (or views) up to INT32_MAX.  An image whose coefficient records could
 * pass 2^32 (6 per byte of the file plus 128 per restart interval: a file with very many short restart intervals, e.g.
 * 8-bit gray with DRI 1 and 10 bytes per interval above about 21 M intervals) gets JPEG_UNSUPPORTED_FEATURE; the
 * other images of the batch still decode.
 * Progressive files are accepted when options has JPEG_SCALE_EIGHTH: like the reference (src/jpeg.inl:4964-4966,
 * JPEGDecodeMCU_P :1819-1884) only the DC coefficients of the first scan are decoded; otherwise that image's status
 * is JPEG_UNSUPPORTED_FEATURE.  With JPEGB200_OPT_PROGRESSIVE in options they are decoded from all of their scans at
 * every scale instead (see there). */
JPEGB200_BATCH *JPEGB200_batchCreate(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes,
                                     int n, int pixel_type, int options);
/* Region-of-interest decode (crop-then-train data loading).  rois: n x {x, y, w, h} in pixels of the OUTPUT image (after
 * scaling, EXIF thumbnail selection and LUMA_ONLY folding), or NULL = whole images (= JPEGB200_batchCreate).  Image i's
 * output is exactly rows y..y+h-1, columns x..x+w-1 of what the same call without rois produces; tight pitch = w * bytes
 * per pixel.
 *   - Any x, y (no MCU or even-pixel alignment); requires 0 <= x, 0 <= y, w >= 1, h >= 1, x + w <= out_w, y + h <= out_h.
 *     An image whose rectangle breaks this gets status JPEG_INVALID_PARAMETER; the others decode normally.
 *   - JPEGB200_batchImageInfo reports out_w, out_h = w, h; JPEGB200_batchOutputBytes, the device arena and
 *     JPEGB200_C_OUTPUT_BYTES follow from that.
 *   - Dithered pixel types: returns NULL (error diffusion runs across the whole image, so the dither of a rectangle is
 *     not a rectangle of the dither).  Every other pixel type, scale and sampling is supported.
 *   - Work: only the MCUs the rectangle touches are transformed and only its pixels are stored; restart intervals that
 *     start below its last MCU row are not walked (JPEGB200_C_SEGMENTS counts the walked ones).  Intervals above it are:
 *     the reference's bit-window phase carries from interval to interval.  (A progressive file decoded with
 *     JPEGB200_OPT_PROGRESSIVE: each scan stops after the rectangle's last MCU row; with views, after the deepest one's.)
 *   - Status follows the reference's crop decode, which parses every MCU row down to the rectangle's last one and no
 *     further: JPEG_DECODE_ERROR exactly when the full decode's first undecodable MCU lies in an MCU row at or above the
 *     last MCU row the rectangle touches; JPEGB200_batchErrMcu then returns that full-image MCU index.  Otherwise the
 *     status is JPEG_SUCCESS and JPEGB200_batchErrMcu returns -1, even if the scan is corrupt further down.  The same
 *     holds for scans without restart markers. */
JPEGB200_BATCH *JPEGB200_batchCreateROI(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes,
                                        int n, int pixel_type, int options, const int32_t *rois);
/* Oriented decode: image i's output is D = T_k(S), S being what the same call without orients produces (after scaling,
 * thumbnail selection and LUMA_ONLY folding, progressive files at 1/8 included), k one of the 8 EXIF transforms:
 *   1 identity, 2 mirror x, 3 rotate 180, 4 mirror y, 5 transpose, 6 rotate 90 clockwise, 7 transverse,
 *   8 rotate 90 counter-clockwise.  For 5-8 out_w and out_h swap.
 * orients[i]: 0 = from the file (JPEG_getOrientation's tag if it is 1-8, identity otherwise: no tag, 0, 9, 255, ...);
 * 1-8 = that transform whatever the file says (a loader composes the EXIF transform with its own random flip);
 * anything else gives that image JPEG_INVALID_PARAMETER.  orients = NULL is JPEGB200_batchCreateROI.
 *   - rois are in the OUTPUT (upright) frame: image i's output is D[y:y+h, x:x+w].  The work skipped and the status rule are
 *     those of JPEGB200_batchCreateROI for the same rectangle in the stored frame (where the scan's MCU rows are): with k = 3
 *     a rectangle at the top of the upright image lies at the bottom of the scan, so almost every restart interval is
 *     walked and an error near the end of the scan is reported.
 *   - Pixels are those of the unrotated decode, bit for bit: the transform is applied by the kernels' stores.
 *   - JPEGB200_batchImageInfo, JPEGB200_batchOutputBytes, the device arena and JPEGB200_C_OUTPUT_BYTES follow the output
 *     frame; the destination rules of JPEGB200_batchSetOutput apply to it unchanged.
 *   - Dithered pixel types and padded output: returns NULL.
 *   - The JPEG_AUTO_ROTATE option bit stays ignored here and in JPEG_decode, as in the reference.
 * Upright sizes before choosing rectangles: create a plain batch (header parse only, no GPU work), read
 * JPEGB200_batchOrientation and JPEGB200_batchImageInfo (swap out_w / out_h for tags 5-8), destroy it, then create the
 * oriented batch. */
JPEGB200_BATCH *JPEGB200_batchCreateOriented(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes,
                                             int n, int pixel_type, int options, const int32_t *rois, const uint8_t *orients);
/* Resized decode (a loader's crop -> flip -> resize in one call).  S_i = what JPEGB200_batchCreateOriented produces for
 * image i with the same rois / orients (after scaling, thumbnail selection and LUMA_ONLY folding); out_sizes[2i], [2i+1] =
 * W, H.  Image i's output is Pillow's Image.resize((W, H), filter) of every byte plane of S_i viewed as [rows, cols, bytes
 * per pixel], bit for bit (PIL/libImaging/Resample.c: double coefficients rounded to 22-bit integers, a horizontal pass
 * into a uint8 intermediate holding only the source rows the vertical pass reads, then the vertical pass; a pass along an
 * axis whose size does not change is skipped, so W, H = S's size gives S).  Crop, then orient, then resize: torchvision's
 * resized_crop on PIL images.  out_sizes = NULL is JPEGB200_batchCreateOriented (filter ignored).
 *   - filter: JPEGB200_RESIZE_BILINEAR, _BICUBIC or _BOX (PIL.Image.Resampling's numbers).  NEAREST is another algorithm
 *     in Pillow; HAMMING and LANCZOS need sin(), whose device rounding is not libm's.
 *   - Pixel types: RGB8888 (in the SSE2-build byte order B,G,R,A too: planes are independent, the 0xFF alpha plane stays
 *     0xFF) and EIGHT_BIT_GRAYSCALE, LUMA_ONLY folding included; every scale, progressive at 1/8, EXIF thumbnails.
 *   - Returns NULL with a message for RGB565 (a 5/6/5 word has no byte planes), dithered types, padded output and any
 *     other filter.  A W or H outside 1..65535 gives that image JPEG_INVALID_PARAMETER; the others decode.
 *   - Status, JPEGB200_batchErrMcu and the restart intervals walked are those of the same ROI / orient plan; an image with
 *     JPEG_DECODE_ERROR gets the resize of what the unresized call stores for it.
 *   - JPEGB200_batchImageInfo reports out_w, out_h = W, H; JPEGB200_batchOutputBytes, the device arena,
 *     JPEGB200_C_OUTPUT_BYTES, the D2H bytes and the destination rules of JPEGB200_batchSetOutput follow W x H.
 *   - Device work: the IDCT stage writes S into library scratch (pooled device memory: S plus the intermediate per image),
 *     then jdk_resize_coeffs / _h / _v; timed in the JPEGB200_T_DITHER slot. */
#define JPEGB200_RESIZE_BILINEAR 2
#define JPEGB200_RESIZE_BICUBIC  3
#define JPEGB200_RESIZE_BOX      4
JPEGB200_BATCH *JPEGB200_batchCreateResized(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                            int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                                            const int32_t *out_sizes /* n x {W, H}; NULL = no resize */, int filter);
/* Tensor output (a model's input tensor, straight from the decode).  U_i = what JPEGB200_batchCreateResized stores for image
 * i with the same rois / orients / out_sizes / filter (crop, orient, resize, every scale, EXIF thumbnail, progressive at
 * 1/8), W x H pixels.  Image i's output is a tensor of C x H x W elements (CHW) or H x W x C (HWC):
 *   - C = 3 for RGB8888: output channel 0 is true red (blue with spec->bgr), 1 green, 2 blue (red with bgr); the library
 *     applies U_i's own byte order (B,G,R,A with the SSE2-build arithmetic at full scale for 4:2:0 and 4:4:4 files, R,G,B,A
 *     otherwise, decided per image), and the alpha byte is dropped.  C = 1 for EIGHT_BIT_GRAYSCALE and LUMA_ONLY folding;
 *     only mean[0] and std[0] are used then.
 *   - Element for byte value x of output channel c: s = (float)x (SCALE_NONE), (float)x / 255.0f (SCALE_DIV255: torchvision
 *     to_tensor) or (float)x * (float)(1.0 / 255) (SCALE_MUL255: torchvision v2 ToDtype(float32, scale=True)); then
 *     y = (s - mean[c]) / std[c], each operation one IEEE float32 rounding (torchvision's Normalize), then round to
 *     nearest even to the dtype (torch's .half() / .bfloat16()).  Bit for bit: the host computes the C x 256 values once per
 *     batch and the kernel only looks them up.  JPEGB200_DT_U8 is a layout conversion: it needs SCALE_NONE, mean 0, std 1.
 *   - Returns NULL with a message for RGB565, dithered types, padded output, an unknown dtype / layout / scale, a std that
 *     is 0 or not finite or a mean that is not finite (over the C channels used), and U8 with any normalization.
 *   - Destinations are device memory only (JPEGB200_batchSetOutputTensor + JPEGB200_batchDecode with JPEGB200_OUT_DEVICE, or
 *     the device arena): batchDecode without JPEGB200_OUT_DEVICE, or a destination that is not device memory of the
 *     context's GPU, fails with a message.  Element (c, y, x) of CHW lies at out + c * plane_stride + y * pitch + x * elt,
 *     element (y, x, c) of HWC at out + y * pitch + (x * C + c) * elt.  Only the tensor's elements are written: not the
 *     pitch padding, not the bytes between planes, not the slot of a rejected image.
 *   - JPEGB200_batchImageInfo reports out_w, out_h = W, H.  JPEGB200_batchOutputBytes = C * H * W * elt with pitch_bytes =
 *     the row bytes (W * elt for CHW, W * C * elt for HWC); the device arena (each tensor tight, 256-byte aligned),
 *     JPEGB200_batchGetDeviceOutput, JPEGB200_batchReadOutput and JPEGB200_C_OUTPUT_BYTES follow from that.
 *   - Status, JPEGB200_batchErrMcu and the restart intervals walked are those of the same call without spec.
 *   - Device work: the pipeline writes U_i into pooled uint8 staging instead of the destination (the IDCT stage, or the
 *     resize's last pass), then one jdk_tensor launch converts every image; timed in the JPEGB200_T_DITHER slot with the
 *     resize.  One launch more than the same call without spec.
 * spec = NULL is JPEGB200_batchCreateResized. */
#define JPEGB200_DT_U8   0
#define JPEGB200_DT_F32  1
#define JPEGB200_DT_F16  2
#define JPEGB200_DT_BF16 3
#define JPEGB200_LAYOUT_CHW 0          /* planar: plane c at out + c * plane_stride, row y at + y * pitch */
#define JPEGB200_LAYOUT_HWC 1          /* interleaved (torch channels_last): pixel x of row y at out + y * pitch + x * C * elt */
#define JPEGB200_SCALE_NONE   0        /* s = (float)x */
#define JPEGB200_SCALE_DIV255 1        /* s = (float)x / 255.0f             (torchvision to_tensor) */
#define JPEGB200_SCALE_MUL255 2        /* s = (float)x * (float)(1.0 / 255)  (torchvision v2 ToDtype(float32, scale=True)) */
typedef struct {
    int32_t dtype, layout, scale, bgr; /* bgr != 0: output channel 0 is blue */
    float mean[3], std[3];             /* per OUTPUT channel: y = (s - mean[c]) / std[c], each step one IEEE float32
                                          rounding, then round-to-nearest-even to dtype (torch's .half() / .bfloat16()) */
} JPEGB200_TensorSpec;
JPEGB200_BATCH *JPEGB200_batchCreateTensor(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                           int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                                           const int32_t *out_sizes, int filter, const JPEGB200_TensorSpec *spec);
/* Destination of image i of a tensor batch (device memory).  pitch: bytes between rows, <= 0 = tight (the row bytes);
 * plane_stride: bytes between the planes of CHW, 0 = pitch * H, ignored for HWC.  Pointer, pitch and plane stride must be
 * multiples of the element size; the pitch must be at least the row bytes and below 2^32, a plane stride at least
 * pitch * H.  Returns 0 with a message, and nothing changed, otherwise.  JPEGB200_batchSetOutput(b, i, out, pitch) on a
 * tensor batch is this call with plane_stride 0. */
int JPEGB200_batchSetOutputTensor(JPEGB200_BATCH *b, int i, void *out, int64_t pitch, int64_t plane_stride);
/* Several views of each file from one entropy walk (multi-crop loaders: SimCLR / MoCo pairs, DINO's global and local crops,
 * FiveCrop / TenCrop).  views[i] >= 1 is the number of views of file i; V = the sum.  The views of file i are the consecutive
 * view indices starting at views[0] + ... + views[i-1].  rois (V x 4), orients (V), out_sizes (V x 2) hold one entry per VIEW,
 * and so do the batch's images from here on: JPEGB200_batchCount returns V and every per-image call (batchImageInfo,
 * batchOutputBytes, batchSetOutput / _Tensor, batchGetDeviceOutput, batchReadOutput, batchErrMcu, batchOrientation, the
 * status of batchWait) takes a view index.  views = NULL is JPEGB200_batchCreateTensor (one view per file).
 *   - The result is that of JPEGB200_batchCreateTensor on the EXPANDED file list (file i repeated views[i] times, in order)
 *     with the same per-view arrays: every output byte (and the bytes left alone), status, batchErrMcu, batchOrientation,
 *     batchImageInfo and batchOutputBytes value, destination rule and refusal.
 *   - Paid once per file: the upload of its bytes, jdk_prescan, the entropy walk (restart intervals down to the deepest last
 *     MCU row among its valid views, or the chunk path of a restart-free scan), jdk_stitch / jdk_patch, the block headers and
 *     coefficient records.  Paid per view: the IDCT / colour stores of its MCU box, the resize and the tensor conversion.
 *   - Counted once per file: JPEGB200_C_COMPRESSED_BYTES, _H2D_BYTES (the per-view descriptors and quantisation tables are
 *     still per view), _SEGMENTS, _BLOCKS, _RECORD_BYTES, _EVENTS and _EVENT_CANDIDATES; the status read-back in
 *     _D2H_BYTES is one descriptor per file.  _OUTPUT_BYTES counts per view.  The window-event overflow of a job
 *     (batchWait) is judged on the candidates counted once per file.
 *   - Status: a file that fails to parse gives its status to all of its views.  A view whose own arguments are invalid
 *     (rectangle outside the output, orientation outside 0-8, W or H outside 1..65535) gets JPEG_INVALID_PARAMETER alone;
 *     the file's other views still decode, and a file without a valid view is not walked.  The file's walk reports its
 *     first undecodable MCU m (no rectangle rule); a view gets JPEG_DECODE_ERROR with batchErrMcu = m when it has no
 *     rectangle or m lies above the end of its last MCU row, else JPEG_SUCCESS and -1 -- the rule of
 *     JPEGB200_batchCreateROI, since a view's walk is a prefix of its file's.
 *   - Returns NULL with a message for any views[i] < 1, V above INT32_MAX, dithered pixel types and padded output. */
JPEGB200_BATCH *JPEGB200_batchCreateViews(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                          const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                          const uint8_t *orients, const int32_t *out_sizes, int filter,
                                          const JPEGB200_TensorSpec *spec);
/* Reduced-size decodes per view, bit-exact with Pillow's Image.draft() (libjpeg-turbo's scale_num / scale_denom = 1 / s):
 * the arguments of JPEGB200_batchCreateViews plus draft, one denominator s per VIEW (1, 2, 4 or 8).  draft = NULL is
 * JPEGB200_batchCreateViews, which forwards here.
 *   - View v with s = draft[v]: its unrotated, uncropped image is libjpeg-turbo's decode at 1 / s, ceil(W / s) x
 *     ceil(H / s) pixels, made with libjpeg's reduced IDCTs (jidctred.c 4x4 / 2x2 / 1x1, and islow where a chroma component
 *     keeps 8x8) and its upsampling at that scale (fancy, none, or replication at 1/8).  rois are in that frame after
 *     orientation; orientation, resize and tensor output then apply unchanged, and batchImageInfo / batchOutputBytes
 *     report the scaled sizes.  s = 1 is byte for byte the JPEGB200_OPT_LIBJPEG output.  Views of one file may use
 *     different scales; the file is still walked once, at full scale.
 *   - Status, batchErrMcu and the walked intervals follow the rules of JPEGB200_batchCreateViews, with each view's MCU box
 *     computed in its scaled frame.
 *   - Needs JPEGB200_OPT_LIBJPEG: a non-NULL draft without it returns NULL with a message.  A value other than 1, 2, 4 or
 *     8 gives that view alone JPEG_INVALID_PARAMETER.  JPEG_SCALE_* stays refused with JPEGB200_OPT_LIBJPEG. */
JPEGB200_BATCH *JPEGB200_batchCreateDraft(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                          const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                          const uint8_t *orients, const int32_t *out_sizes, int filter,
                                          const JPEGB200_TensorSpec *spec, const uint8_t *draft);
/* Pillow's choice of s for draft(mode, (req_w, req_h)) on a W x H file: k = min(W / req_w, H / req_h) (integer division),
 * then the largest of 8, 4, 2, 1 that is at most k, else 1.  A request of 0 (where Pillow would divide by zero) gives 1. */
int JPEGB200_draftScale(int width, int height, int req_w, int req_h);
/* Resize with a source box and a reducing gap, bit-exact with Pillow's Image.resize((W, H), filter, box=, reducing_gap=)
 * (what Image.thumbnail() runs after its draft): the arguments of JPEGB200_batchCreateDraft plus, per VIEW,
 * boxes[4 v .. 4 v + 3] = x0, y0, x1, y1 (doubles, fractional allowed) and reducing_gaps[v] (0 = Pillow's None).
 *   - S_v is what JPEGB200_batchCreateDraft stores for view v without out_sizes (crop, then orientation, at its draft
 *     scale).  View v's output is Pillow's resize of every byte plane of S_v to out_sizes[v] with that box and gap:
 *     with a gap, the reduce (Image.reduce) by int(box extent / out / gap) or 1 per axis of the box widened by the
 *     filter's support, the box carried into the reduced frame; Pillow's vertical-pass-first rule for sources more than
 *     100 times taller than wide; the C resize's passes for any box that does not start at 0 and end at the output size.
 *   - boxes = NULL means (0, 0, S_w, S_h) and reducing_gaps = NULL no reduce; with both NULL this is
 *     JPEGB200_batchCreateDraft, which forwards here.  Status, batchErrMcu, the walked intervals and the destination rules
 *     are those of the same call without boxes and gaps.
 *   - Filters are those of the resize (BILINEAR, BICUBIC, BOX).  Boxes or gaps without out_sizes return NULL with a message.
 *     A view whose box or gap Pillow refuses (a box value that is not finite, a negative offset, past S_v or with a negative
 *     extent, checked on the box as float; gap < 1), whose reduce would be empty or reduce boxes of 2^23 pixels or more,
 *     gets JPEG_INVALID_PARAMETER alone.  A box past S_v is refused even where Pillow's reduce would carry it inside the
 *     reduced image.
 *   - The reduce and the boxed coefficient tables are timed in the JPEGB200_T_DITHER slot with the resize; the reduced
 *     image counts in the one-call path's scratch bound. */
JPEGB200_BATCH *JPEGB200_batchCreateBox(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                        const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                        const uint8_t *orients, const int32_t *out_sizes, int filter,
                                        const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                        const double *reducing_gaps);
/* Pillow's Image.thumbnail((req_w, req_h), BICUBIC, reducing_gap) decision for a W x H JPEG (reducing_gap 0 = None):
 * preserve_aspect_ratio (floor or ceil of the exact side, whichever keeps W / H closer, floor on a tie, at least 1), the
 * draft scale of the request int(req * gap) (JPEGB200_draftScale; 1 without a gap) and the box (0, 0, W / s, H / s).
 * Writes *draft, *out_w x *out_h and box[4] such that JPEGB200_batchCreateBox with draft, out_sizes, boxes and reducing_gaps
 * (the same gap) decodes the file's thumbnail.  Returns JPEGB200_THUMB_RESIZE; JPEGB200_THUMB_DRAFT when the draft decode is
 * already the final size (Pillow stores it without a resize; box is then the whole drafted image); JPEGB200_THUMB_NONE when
 * the request covers the file (Pillow leaves it alone: draft 1, the file's size, the whole image); 0 for a size or request
 * below 1, a gap below 1 that is not 0, or a NULL output. */
#define JPEGB200_THUMB_RESIZE 1
#define JPEGB200_THUMB_DRAFT  2
#define JPEGB200_THUMB_NONE   3
int JPEGB200_thumbnailPlan(int width, int height, int req_w, int req_h, double reducing_gap, int *draft, int *out_w, int *out_h,
                           double *box);
/* Per-view colour operations, bit-exact with torchvision's ColorJitter (adjust_brightness / _contrast / _saturation / _hue),
 * RandomGrayscale and RandomSolarize on a PIL image (Pillow 12's arithmetic): the arguments of JPEGB200_batchCreateBox plus
 * color_ops, V x JPEGB200_COLOR_MAX_OPS entries, row v holding view v's operations in order and ending at the first op 0.
 *   - F_v is what JPEGB200_batchCreateBox stores for view v (crop, orientation, draft, box, reduce, resize), as uint8 pixels.
 *     View v's operations run on F_v in the order given, before the tensor conversion, on true R, G, B (the byte order of
 *     an RGB8888 view, R, G, B, A or B, G, R, A, is that of the same call; the alpha byte is left as it is):
 *       BRIGHTNESS f  ImageEnhance.Brightness: c = blend(0, c, f)
 *       CONTRAST f    ImageEnhance.Contrast: c = blend(m, c, f), m = int(sum of L over the current image / (W H) + 0.5)
 *       SATURATION f  ImageEnhance.Color: c = blend(L, c, f)
 *       HUE h         adjust_hue: Pillow's convert("HSV"), H += uint8(int32(h * 255)) mod 256, convert("RGB").  The HSV round
 *                     trip itself changes pixels, so h = 0 is not the identity (it is torchvision's adjust_hue(img, 0)).
 *       GRAYSCALE     to_grayscale(img, 3): R = G = B = L (arg ignored)
 *       SOLARIZE t    ImageOps.solarize(img, t): c < t ? c : 255 - c, t compared as a double
 *       GAUSSIAN_BLUR r  img.filter(ImageFilter.GaussianBlur(r)) (Pillow's extended box filter, three passes per direction,
 *                     edges replicated; DESIGN.md 4.2.10).  R, G and B are blurred independently, so the byte order does
 *                     not matter; the alpha byte is kept.  r = 0 is the identity and is dropped; r < 0 gives the bytes of
 *                     |r|.  Flips commute with the blur (symmetric window, clamped edges), so a recipe that blurs before
 *                     its flip gets the same bytes from the orientation in the pixel stores.
 *     with L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16 (convert("L")) and blend(a, b, f) = Image.blend: t = (float)a +
 *     (float)f * (float)(b - a) in float32; (uint8)t for 0 <= f <= 1, else clamped to 0 .. 255 and truncated.
 *   - 8-bit gray output (EIGHT_BIT_GRAYSCALE, JPEG_LUMA_ONLY) is a Pillow "L" image: brightness, contrast (m over the bytes),
 *     solarize and the blur apply; saturation, hue and grayscale leave it unchanged, as in Pillow and torchvision.
 *   - color_ops = NULL is JPEGB200_batchCreateBox, which forwards here.  A view whose row is empty stores F_v.  Factor 1
 *     and a solarize threshold above 255 store F_v too.  Status, batchErrMcu, the walked intervals, sizes, output bytes and
 *     the destination rules are those of the same call without operations; only the image's own bytes are rewritten.
 *   - Returns NULL with a message for RGB565, dithered pixel types and padded output when any view has an operation.  A view
 *     with an unknown op, an argument that is not finite, HUE outside [-0.5, 0.5] or a blur radius whose float32 magnitude
 *     is 2^31 or more (|r| >= 2147483584; Pillow's box radius overflows there) gets JPEG_INVALID_PARAMETER alone.
 *     Negative factors are accepted: Pillow extrapolates.
 *   - Device work: the operations run in place on each view's uint8 result (the destination, the arena or the tensor
 *     staging).  A view's list is cut at each CONTRAST and each GAUSSIAN_BLUR; at cut index s (0 = the list's start) the
 *     call makes, over all views, the blur pair jdk_blur_h + jdk_blur_v when some view blurs there, then one jdk_color
 *     launch when some view has a per-pixel operation before its next cut or a CONTRAST at it (that launch sums L per view,
 *     exact in 64 bits).  Without blurs that is 1 + the most CONTRAST operations of any view; none when no view has an
 *     operation.  The blur pair goes through a scratch copy of the blurred views (w x h x 4 or 1 bytes each), counted in the
 *     one-call path's per-job scratch bound.  Timed in the JPEGB200_T_DITHER slot, counted in JPEGB200_C_LAUNCHES. */
#define JPEGB200_COLOR_BRIGHTNESS 1
#define JPEGB200_COLOR_CONTRAST   2
#define JPEGB200_COLOR_SATURATION 3
#define JPEGB200_COLOR_HUE        4
#define JPEGB200_COLOR_GRAYSCALE  5
#define JPEGB200_COLOR_SOLARIZE   6
#define JPEGB200_COLOR_GAUSSIAN_BLUR 16
/* The auto-augment operations of torchvision's RandAugment / TrivialAugmentWide / AutoAugment on a PIL image (the arg is the
 * magnitude torchvision's _apply_op receives; Brightness / Color / Contrast / Solarize / Identity are the ops above):
 *       SHARPNESS f    F.adjust_sharpness(img, f): blend(SMOOTH(img), img, f), SMOOTH's border pixels unchanged
 *       POSTERIZE b    F.posterize(img, b), b an integer 0 .. 8
 *       AUTOCONTRAST   F.autocontrast(img), per channel (arg ignored)
 *       EQUALIZE       F.equalize(img), per channel (arg ignored)
 *       INVERT         F.invert(img) (arg ignored)
 *       SHEAR_X m, SHEAR_Y m, TRANSLATE_X m, TRANSLATE_Y m (int(m) pixels), ROTATE m (degrees, counter-clockwise):
 *                      _apply_op(img, "ShearX" .. "Rotate", m, NEAREST, fill=None); the view keeps its size, pixels from
 *                      outside the image are 0 (alpha kept).
 *   They apply to gray views too, on the one channel.  A posterize argument that is not an integer in 0 .. 8, or a
 *   geometric op on a view wider or taller than 1024 pixels (the sizes pinned against Pillow) or whose fixed-point mapping
 *   does not fit 32 bits, gives that view JPEG_INVALID_PARAMETER.  The list is also cut at each SHARPNESS, AUTOCONTRAST,
 *   EQUALIZE and geometric op: at such a cut index the call makes jdk_augment + jdk_augment_copy when some view sharpens
 *   or moves pixels there (through the blur's scratch copy).  A cut index where some view posterizes, inverts, applies an
 *   AUTOCONTRAST / EQUALIZE or counts the histogram for one runs jdk_color_lut in place of jdk_color: the launch before an
 *   AUTOCONTRAST or EQUALIZE counts per-view histograms (768 64-bit counts per op, counted in the one-call path's scratch
 *   bound), from which the next one builds the LUT.  Lists without these ops make the same launches as before.
 *   DESIGN.md 4.2.11. */
#define JPEGB200_COLOR_SHARPNESS    20
#define JPEGB200_COLOR_POSTERIZE    21
#define JPEGB200_COLOR_AUTOCONTRAST 22
#define JPEGB200_COLOR_EQUALIZE     23
#define JPEGB200_COLOR_INVERT       24
#define JPEGB200_COLOR_SHEAR_X      25
#define JPEGB200_COLOR_SHEAR_Y      26
#define JPEGB200_COLOR_TRANSLATE_X  27
#define JPEGB200_COLOR_TRANSLATE_Y  28
#define JPEGB200_COLOR_ROTATE       29
/* A filter flag OR'd into one of the five geometric codes (25 .. 29), e.g. JPEGB200_COLOR_ROTATE | JPEGB200_COLOR_BILINEAR:
 * the op is _apply_op(img, "ShearX" .. "Rotate", m, BILINEAR or BICUBIC, fill=None) instead, the same argument, size, fill
 * and refusals (a view side above 1024, a non-finite argument).  R, G and B are resampled on their own; gray views too.
 * Both flags together, a flag on any other code or on its own is an unknown op (that view gets JPEG_INVALID_PARAMETER).
 * At a cut index where some view resamples, the call adds jdk_augment_rs, which writes the view's scratch copy, and the
 * jdk_augment_copy that copies it back (one copy launch serves the NEAREST and sharpness views there too).
 * DESIGN.md 4.2.12. */
#define JPEGB200_COLOR_BILINEAR     0x100
#define JPEGB200_COLOR_BICUBIC      0x200
/* Pillow's Image.transform(size, AFFINE or PERSPECTIVE, data, resample, fillcolor) on the view's final image, the size
 * kept: torchvision's RandomAffine, RandomRotation (expand=False) and RandomPerspective on a PIL image (jpegdec_b200's
 * geometric_ops draws them).  Only through JPEGB200_batchCreateWarp / JPEGB200_decodeBatchWarp, whose warp_args entry
 * (v, k) holds op (v, k)'s data (6 coefficients for AFFINE, 8 for PERSPECTIVE) and fill.  A bare code is NEAREST; OR in
 * JPEGB200_COLOR_BILINEAR or _BICUBIC for those filters.  R, G and B are warped on their own; gray views too (fill[0]).
 * Fill values are clamped to 0 .. 255, as Pillow clamps them, and land in the view's own byte order; the alpha byte of a
 * filled RGB8888 pixel is 0xFF.  A view gets JPEG_INVALID_PARAMETER for a non-finite coefficient, both filter flags, a
 * side above 1024 pixels (the sizes pinned against Pillow), or a NEAREST affine with b or d non-zero outside Pillow's 16.16
 * fixed-point range: |x a + y b + c| or |x d + y e + f| at least 32768 at a corner (x = 0 or w, y = 0 or h) of the view
 * (Pillow switches to another form there, which is not pinned).  NEAREST AFFINE with b = d = 0
 * (scale and translate only) follows Pillow's own path for that case.  Through the Color calls both codes are unknown ops.
 * At a cut index where some view warps, the call adds jdk_warp, which writes the view's scratch copy, and the shared
 * jdk_augment_copy.  DESIGN.md 4.2.13. */
#define JPEGB200_COLOR_AFFINE       40
#define JPEGB200_COLOR_PERSPECTIVE  41
/* The JPEG round trip: Pillow's img.save(buf, "JPEG", quality=q) then Image.open(buf), which is torchvision's
 * v2.functional.jpeg(img, q) on a PIL image and on a uint8 tensor alike (jpegdec_b200's jpeg_ops draws v2.JPEG's q).
 *       JPEG q       an RGB view is compressed as Pillow compresses an "RGB" image -- YCbCr, 4:2:0, the baseline tables of
 *                    quality q, islow forward DCT -- and decoded as libjpeg-turbo decodes by default (islow, fancy
 *                    upsampling); a gray view is an "L" image, one component with the luminance table
 *       JPEG_444 q   the same with subsampling=0 (4:4:4)
 *       JPEG_422 q   the same with subsampling=1 (4:2:2)
 *   R, G, B are taken in the view's byte order and the alpha byte is kept.  No file is made: the entropy coding is lossless,
 *   so the quantized coefficients go straight back through the decoder's arithmetic.  A q that is not finite or not an
 *   integer in 1 .. 100 gives that view JPEG_INVALID_PARAMETER alone; any view size is accepted (sides above 65 500,
 *   which libjpeg's encoder and so Pillow's save refuse, get the same arithmetic).  The list is cut at each
 *   JPEG op, as at a blur: the ops before it see the pixels before compression, those after it the decoded pixels.  At a
 *   cut index where some view compresses, the call makes jdk_jq_fwd (one thread per 8 x 8 block: the forward half and the
 *   inverse DCT) over those views, then on RGB output jdk_jq_color (upsampling and colour conversion, in place); a gray
 *   view's blocks are written back in place by jdk_jq_fwd.  The decoded sample planes of an RGB view (its MCUs x blocks per
 *   MCU x 64 bytes) take the blur's scratch, counted in the one-call path's per-job scratch bound.  Lists without these
 *   ops make the same launches as before.  DESIGN.md 4.2.15. */
#define JPEGB200_COLOR_JPEG         31
#define JPEGB200_COLOR_JPEG_444     32
#define JPEGB200_COLOR_JPEG_422     33
#define JPEGB200_COLOR_MAX_OPS    8
typedef struct {
    int32_t op;                        /* JPEGB200_COLOR_*, 0 = end of the view's list */
    double arg;                        /* factor, hue shift (-0.5 .. 0.5), solarize threshold, blur radius or magnitude */
} JPEGB200_ColorOp;
/* the arguments of an AFFINE or PERSPECTIVE op */
typedef struct {
    double coeffs[8];                  /* Pillow's data: a, b, c, d, e, f (AFFINE) and g, h (PERSPECTIVE); the rest unread */
    int32_t fill[3];                   /* true R, G, B (a gray view uses fill[0]), each clamped to 0 .. 255 */
} JPEGB200_WarpArgs;
/* Image.rotate(angle, center=center)'s matrix for a w x h image (center NULL = (w / 2, h / 2)): angle % 360 as Python takes
 * it, the rotation rounded to 15 decimals, the centre kept; the AFFINE data of RandomRotation's draw.  0 for mat NULL. */
int JPEGB200_rotateMatrix(double angle, int w, int h, const double *center, double mat[6]);
JPEGB200_BATCH *JPEGB200_batchCreateColor(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                          const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                          const uint8_t *orients, const int32_t *out_sizes, int filter,
                                          const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                          const double *reducing_gaps, const JPEGB200_ColorOp *color_ops);
/* The same with the AFFINE / PERSPECTIVE arguments: warp_args has V x JPEGB200_COLOR_MAX_OPS entries, parallel to
 * color_ops; entry (v, k) is read only when op (v, k) is AFFINE or PERSPECTIVE.  warp_args = NULL is
 * JPEGB200_batchCreateColor, which forwards here. */
JPEGB200_BATCH *JPEGB200_batchCreateWarp(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                         const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                         const uint8_t *orients, const int32_t *out_sizes, int filter,
                                         const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                         const double *reducing_gaps, const JPEGB200_ColorOp *color_ops,
                                         const JPEGB200_WarpArgs *warp_args);
/* Crop after the resize: torchvision's evaluation preset (Resize -> CenterCrop), FiveCrop, TenCrop and RandomCrop.  The
 * arguments of JPEGB200_batchCreateWarp plus windows: V x {x, y, w, h}, one per view (windows = NULL is
 * JPEGB200_batchCreateWarp, which forwards here).  Let R_v be what the same call without windows has after its resize and
 * before its colour list (rectangle, orientation, draft, box / reduce, resize; uint8).  View v is then Pillow's
 * R_v.crop((x, y, x + w, y + h)) of every byte plane: the window may reach past R_v on any side or lie wholly outside it,
 * and its pixels outside R_v are 0 (RGB8888: R = G = B = 0, alpha 0xFF; gray 0).  Without out_sizes R_v is the unresized
 * image itself, so a window is a rectangle that may pad.  The colour list then runs on the w x h window, and the tensor
 * conversion follows; JPEGB200_batchImageInfo, _batchOutputBytes, the arena, JPEGB200_C_OUTPUT_BYTES and the tensor shape
 * follow w x h.  A w or h outside 1..65535 gives that view alone JPEG_INVALID_PARAMETER; RGB565, dithered pixel types and
 * padded output return NULL, as for out_sizes.
 * The resize reads only the window's support: the rectangle of the unresized image from the first in-image output's
 * first tap to the last one's last tap per resampled axis (the window's in-image span along an axis Pillow does not
 * resample; 1 x 1 at the origin when the window reads no pixel).  The view decodes that rectangle alone, through the
 * region-of-interest decode, inside its own rois rectangle.  So its status and JPEGB200_batchErrMcu follow the
 * JPEGB200_batchCreateROI rule for the support rectangle: a corrupt scan below the support leaves the view at JPEG_SUCCESS,
 * and restart intervals below it are not walked.  A boxed view (boxes or reducing_gaps) decodes all of its rectangle.
 * The passes (which axes, vertical first) are Pillow's choice for the full sizes, so the bytes are those of the full
 * resize.  DESIGN.md 4.2.16. */
JPEGB200_BATCH *JPEGB200_batchCreateWindow(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                           const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                           const uint8_t *orients, const int32_t *out_sizes, int filter,
                                           const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                           const double *reducing_gaps, const JPEGB200_ColorOp *color_ops,
                                           const JPEGB200_WarpArgs *warp_args, const int32_t *windows);
void JPEGB200_batchDestroy(JPEGB200_BATCH *b);
int JPEGB200_batchCount(JPEGB200_BATCH *b);
/* per-image facts after batchCreate: status is JPEG_SUCCESS or the open() error the reference would give */
int JPEGB200_batchImageInfo(JPEGB200_BATCH *b, int i, int32_t *width, int32_t *height, int32_t *subsample,
                            int32_t *out_w, int32_t *out_h, int32_t *status);
/* bytes needed for a tightly packed output of image i (out_h rows of out_pitch bytes) */
int64_t JPEGB200_batchOutputBytes(JPEGB200_BATCH *b, int i, int64_t *pitch_bytes);
/* Destination for image i.  Device pointer if the batch is decoded with JPEGB200_OUT_DEVICE, else host
 * (pinned recommended).  pitch_bytes <= 0 -> tight (the row bytes of JPEGB200_batchOutputBytes).  Returns 0, with a message
 * and nothing changed, for a pitch below the row bytes or above 2^32 - 1.  The decode writes out_h rows of row bytes at
 * out + y * pitch and nothing else: not the pitch padding, not the slot of a rejected image.  (For 1-bit dither with a
 * padded width that is not a multiple of 8, the half-covered last byte of a row is not stored and is not defined.)
 * Device outputs: pointer and pitch must be multiples of the pixel store size (2 RGB565, 4 RGB8888, 1 gray / dithered);
 * JPEGB200_batchDecode returns 0 before enqueueing anything otherwise. */
int JPEGB200_batchSetOutput(JPEGB200_BATCH *b, int i, void *out, int64_t pitch_bytes);
/* Let the library own a device output arena (tight images back to back, 256-B aligned). */
int JPEGB200_batchAllocDeviceOutput(JPEGB200_BATCH *b);
int JPEGB200_batchGetDeviceOutput(JPEGB200_BATCH *b, int i, void **devptr, int64_t *pitch_bytes);
int JPEGB200_batchReadOutput(JPEGB200_BATCH *b, int i, void *host_dst); /* synchronous D2H of one image from the arena */
int JPEGB200_batchErrMcu(JPEGB200_BATCH *b, int i);                      /* first undecodable MCU of image i, -1 if none */
/* Any batch, right after creation: exif_tag = the file's EXIF Orientation tag (0 if it has none), applied = the transform
 * the decode applies (1-8; 1 for a batch created without orients). */
int JPEGB200_batchOrientation(JPEGB200_BATCH *b, int i, int32_t *exif_tag, int32_t *applied);
/* dither needs no extra buffers from the caller: packed rows are written to the output. */

int JPEGB200_batchUpload(JPEGB200_BATCH *b);            /* H2D: compressed bytes + descriptors (async) */
int JPEGB200_batchDecode(JPEGB200_BATCH *b, int flags); /* kernel launches (async) */
int JPEGB200_batchDownload(JPEGB200_BATCH *b);          /* D2H of pixels for host outputs (async) */
int JPEGB200_batchWait(JPEGB200_BATCH *b, int32_t *status /* n entries, may be NULL */);
int JPEGB200_batchGetTimings(JPEGB200_BATCH *b, float *ms /* JPEGB200_NUM_TIMINGS */);
int JPEGB200_batchGetCounters(JPEGB200_BATCH *b, int64_t *counters /* JPEGB200_NUM_COUNTERS */);
void *JPEGB200_batchStream(JPEGB200_BATCH *b);          /* cudaStream_t the job runs on */

/* One call for a whole batch of ANY size: create + upload + decode + (download) + wait + destroy.
 * outs[i]: destination (host, or the caller's device memory with JPEGB200_OUT_DEVICE); pitches may be NULL (tight).
 * The batch is run as a pipeline of jobs on separate streams: with host outputs the pixels of one job cross PCIe while the
 * next job's kernels run; with device outputs a job holds at most 192 MiB of compressed bytes, which bounds the transient
 * device memory however large the batch is (the reference equivalent is a loop of JPEG_openRAM + JPEG_decode,
 * src/JPEGDEC.cpp:157-224, which streams any input through a 2 KB window, src/jpeg.inl:1544-1566).
 * Destinations follow JPEGB200_batchSetOutput: pitch at least the row bytes and below 2^32; device pointers and pitches
 * multiples of the pixel store size.  A destination that breaks this fails the call (0) with a message naming the image
 * index (in this call), the pitch and the row bytes.  Only each image's rows are written, except that host buffers laid out
 * like the device arena (image i at outs[0] + its 256-byte-aligned arena offset, tight pitches) are filled by one copy that
 * also writes the gaps between images.
 * Returns 1 = all images decoded, 2 = some images failed (see status[]), 0 = call failed. */
int JPEGB200_decodeBatch(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                         int pixel_type, int options, void *const *outs, const int64_t *pitches,
                         int flags, int32_t *status);
/* The same with a region of interest per image (rois: n x {x, y, w, h}, semantics of JPEGB200_batchCreateROI; NULL = whole
 * images).  outs[i] receives h rows of w pixels. */
int JPEGB200_decodeBatchROI(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                            int pixel_type, int options, const int32_t *rois, void *const *outs,
                            const int64_t *pitches, int flags, int32_t *status);
/* The same with an orientation per image (orients: n entries, semantics of JPEGB200_batchCreateOriented; NULL = none).
 * outs[i] receives the output-frame image (or rectangle of it). */
int JPEGB200_decodeBatchOriented(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                 int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                                 void *const *outs, const int64_t *pitches, int flags, int32_t *status);
/* The same with a resize per image (out_sizes: n x {W, H}, filter: semantics of JPEGB200_batchCreateResized; NULL = none).
 * outs[i] receives H rows of W pixels.  Each job also holds at most 1 GiB of resize scratch (the unresized outputs plus
 * the intermediates), or one image if a single image needs more, so the transient device memory of the call stays
 * bounded however many images it decodes: each job in flight holds at most that scratch plus, with device outputs, 192 MiB
 * of compressed bytes and their coefficient records. */
int JPEGB200_decodeBatchResized(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                                const int32_t *out_sizes, int filter, void *const *outs, const int64_t *pitches,
                                int flags, int32_t *status);
/* The same into tensors (spec: semantics of JPEGB200_batchCreateTensor; NULL = JPEGB200_decodeBatchResized).  With spec,
 * flags must hold JPEGB200_OUT_DEVICE and outs[i] are device tensors with pitches[i] (NULL or <= 0 = tight) and
 * plane_strides[i] (NULL or 0 = pitch * H) under the rules of JPEGB200_batchSetOutputTensor.  The 1 GiB of scratch per
 * job counts the uint8 staging of the tensors too. */
int JPEGB200_decodeBatchTensor(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                               int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                               const int32_t *out_sizes, int filter, const JPEGB200_TensorSpec *spec, void *const *outs,
                               const int64_t *pitches, const int64_t *plane_strides, int flags, int32_t *status);
/* The same with several views per file (views: n per-file counts, semantics of JPEGB200_batchCreateViews; NULL =
 * JPEGB200_decodeBatchTensor).  rois, orients, out_sizes, outs, pitches, plane_strides and status hold one entry per view.
 * Jobs are cut at file boundaries only: the views of one file are always decoded by one job.  The per-job image cap, the
 * host-output job re-plan for small images and the 1 GiB of scratch per job count views; a file whose views alone need more
 * scratch gets a job of its own.  Error messages name the view index in this call. */
int JPEGB200_decodeBatchViews(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                              const int32_t *views, int pixel_type, int options, const int32_t *rois,
                              const uint8_t *orients, const int32_t *out_sizes, int filter,
                              const JPEGB200_TensorSpec *spec, void *const *outs, const int64_t *pitches,
                              const int64_t *plane_strides, int flags, int32_t *status);
/* The same with a draft scale per view (semantics of JPEGB200_batchCreateDraft; NULL = JPEGB200_decodeBatchViews, which
 * forwards here).  The 1 GiB of scratch per job counts each view's sample planes at its own scale. */
int JPEGB200_decodeBatchDraft(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                              const int32_t *views, int pixel_type, int options, const int32_t *rois,
                              const uint8_t *orients, const int32_t *out_sizes, int filter,
                              const JPEGB200_TensorSpec *spec, const uint8_t *draft, void *const *outs, const int64_t *pitches,
                              const int64_t *plane_strides, int flags, int32_t *status);
/* The same with a box and a reducing gap per view (semantics of JPEGB200_batchCreateBox; both NULL =
 * JPEGB200_decodeBatchDraft, which forwards here).  The reduced images count in the 1 GiB of scratch per job. */
int JPEGB200_decodeBatchBox(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n, const int32_t *views,
                            int pixel_type, int options, const int32_t *rois, const uint8_t *orients, const int32_t *out_sizes,
                            int filter, const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                            const double *reducing_gaps, void *const *outs, const int64_t *pitches, const int64_t *plane_strides,
                            int flags, int32_t *status);
/* The same with colour operations per view (color_ops: V x JPEGB200_COLOR_MAX_OPS, semantics of JPEGB200_batchCreateColor;
 * NULL = JPEGB200_decodeBatchBox, which forwards here).  Without blurs the jobs are those of the call without operations
 * (8 bytes of scratch per view and contrast); a blurred view's scratch copy counts in the per-job scratch bound. */
int JPEGB200_decodeBatchColor(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                              const int32_t *views, int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                              const int32_t *out_sizes, int filter, const JPEGB200_TensorSpec *spec, const uint8_t *draft,
                              const double *boxes, const double *reducing_gaps, const JPEGB200_ColorOp *color_ops,
                              void *const *outs, const int64_t *pitches, const int64_t *plane_strides, int flags,
                              int32_t *status);
/* The same with the AFFINE / PERSPECTIVE arguments (warp_args: semantics of JPEGB200_batchCreateWarp; NULL =
 * JPEGB200_decodeBatchColor, which forwards here).  A warped view's scratch copy counts in the per-job scratch bound. */
int JPEGB200_decodeBatchWarp(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                             const int32_t *views, int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                             const int32_t *out_sizes, int filter, const JPEGB200_TensorSpec *spec, const uint8_t *draft,
                             const double *boxes, const double *reducing_gaps, const JPEGB200_ColorOp *color_ops,
                             const JPEGB200_WarpArgs *warp_args, void *const *outs, const int64_t *pitches,
                             const int64_t *plane_strides, int flags, int32_t *status);
/* The same with a window per view (semantics of JPEGB200_batchCreateWindow; NULL = JPEGB200_decodeBatchWarp, which forwards
 * here).  The per-job scratch bound counts each view's support, not its whole unresized image. */
int JPEGB200_decodeBatchWindow(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                               const int32_t *views, int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                               const int32_t *out_sizes, int filter, const JPEGB200_TensorSpec *spec, const uint8_t *draft,
                               const double *boxes, const double *reducing_gaps, const JPEGB200_ColorOp *color_ops,
                               const JPEGB200_WarpArgs *warp_args, const int32_t *windows, void *const *outs,
                               const int64_t *pitches, const int64_t *plane_strides, int flags, int32_t *status);
/* JPEGB200_NUM_COUNTERS counters summed over the jobs of the last JPEGB200_decodeBatch on this context */
int JPEGB200_lastCallCounters(JPEGB200_CTX *ctx, int64_t *counters);
/* CUDA-event stage times (JPEGB200_NUM_TIMINGS, ms) summed over those jobs, and how many jobs there were.  Jobs overlap
 * on the GPU unless the pipeline depth is 1, so the sums are an upper bound of the stage's share of the call. */
int JPEGB200_lastCallTimings(JPEGB200_CTX *ctx, float *ms, int *jobs);
/* jobs JPEGB200_decodeBatch keeps in flight (0 = default: 6 with host outputs, 3 with device outputs; 1 = strictly serial) */
int JPEGB200_setPipelineDepth(JPEGB200_CTX *ctx, int jobs_in_flight);

/* ---- shared-table blob (multi-GPU: rank 0 exports, NCCL broadcast, other ranks import) ---- */
#define JPEGB200_TABLE_BLOB_BYTES (10496 * 2 + 3 * 64 * 2 + 16)
int JPEGB200_exportTables(const uint8_t *jpeg, int size, uint8_t *blob /* JPEGB200_TABLE_BLOB_BYTES */);
int JPEGB200_setSharedTables(JPEGB200_CTX *ctx, const uint8_t *blob);
int JPEGB200_sharedTableHits(JPEGB200_CTX *ctx);

#ifdef __cplusplus
}
#endif
#endif /* JPEGDEC_B200_H */
