/*
 * jd_api.c -- the JPEGDEC C API (include/JPEGDEC.h) on top of the batch pipeline.
 *
 * Boundary being replaced (reference file:line):
 *   JPEG_openRAM / JPEG_openFile / getters / setters ... src/jpeg.inl:564-738
 *   JPEG_decode / JPEG_decodeDither -> DecodeJPEG ....... src/jpeg.inl:655-668, :4946-5357
 *
 * decode() = one-image batch on the GPU (whole MCU-aligned frame into a pinned staging
 * buffer) followed by a host replay of the reference's *delivery* rules: MCU skipping for
 * crop, draw-callback batching (iMCUCount), iWidth / iWidthUsed / iHeight trimming, the DMA
 * ping-pong pointer, framebuffer pitch = crop width.  Pixels are never computed on the host.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include "jd_internal.h"

/* One context per (device, arithmetic build), created on first use.  g_lock guards this table and the staging pool; the GPU
 * work of a decode holds only its context's lock (a context is driven by one thread at a time); the host replay of the
 * delivery rules -- which runs the user's callback -- holds no lock at all, so a callback may decode another image and
 * decodes on different GPUs do not serialise each other (the reference is re-entrant per handle, SURVEY.md 8b). */
#define JD_MAX_DEVICES 64
static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;
static JPEGB200_CTX *g_ctx[JD_MAX_DEVICES][2];
static pthread_mutex_t g_ctx_lock[JD_MAX_DEVICES][2];
static int g_ctx_lock_init;

/* pinned staging frames, recycled (allocating pinned memory costs far more than a small decode) */
#define JD_STAGE_SLOTS 8
static struct { uint8_t *p; size_t bytes; } g_stage[JD_STAGE_SLOTS];

static uint8_t *stage_get(size_t need, size_t *got)
{
    uint8_t *p = NULL;
    pthread_mutex_lock(&g_lock);
    for (int i = 0; i < JD_STAGE_SLOTS; i++)
        if (g_stage[i].p && g_stage[i].bytes >= need) { p = g_stage[i].p; *got = g_stage[i].bytes; g_stage[i].p = NULL; break; }
    pthread_mutex_unlock(&g_lock);
    if (p) return p;
    *got = need + (1u << 20);
    return (uint8_t *)JPEGB200_hostAlloc(*got);
}

static void stage_put(uint8_t *p, size_t bytes)
{
    if (!p) return;
    pthread_mutex_lock(&g_lock);
    int slot = -1;
    for (int i = 0; i < JD_STAGE_SLOTS; i++) {
        if (!g_stage[i].p) { slot = i; break; }
        if (slot < 0 || g_stage[i].bytes < g_stage[slot].bytes) slot = i;
    }
    uint8_t *drop = NULL;
    if (g_stage[slot].p) { if (g_stage[slot].bytes >= bytes) { drop = p; p = NULL; } else drop = g_stage[slot].p; }
    if (p) { g_stage[slot].p = p; g_stage[slot].bytes = bytes; }
    pthread_mutex_unlock(&g_lock);
    if (drop) JPEGB200_hostFree(drop);
}

extern int JPEGB200_currentDevice(void);

/* returns the context and its lock for (device, arith); device < 0 = the calling thread's current CUDA device */
static JPEGB200_CTX *get_ctx(int device, int arith, pthread_mutex_t **lock)
{
    if (device < 0) device = JPEGB200_currentDevice();
    if (device < 0 || device >= JD_MAX_DEVICES) return NULL;
    const int a = arith ? 1 : 0;
    pthread_mutex_lock(&g_lock);
    if (!g_ctx_lock_init) {
        for (int d = 0; d < JD_MAX_DEVICES; d++) { pthread_mutex_init(&g_ctx_lock[d][0], NULL); pthread_mutex_init(&g_ctx_lock[d][1], NULL); }
        g_ctx_lock_init = 1;
    }
    if (!g_ctx[device][a]) g_ctx[device][a] = JPEGB200_create(device, arith);
    JPEGB200_CTX *c = g_ctx[device][a];
    pthread_mutex_unlock(&g_lock);
    *lock = &g_ctx_lock[device][a];
    return c;
}

static void fill_from_info(JPEGIMAGE *p, const JDInfo *inf)
{
    p->iWidth = p->iCropCX = inf->width;
    p->iHeight = p->iCropCY = inf->height;
    p->iCropX = p->iCropY = 0;
    p->ucBpp = (uint8_t)inf->bpp;
    p->ucSubSample = (uint8_t)inf->subsample;
    p->ucMode = (uint8_t)inf->mode;
    p->ucNumComponents = (uint8_t)inf->ncomp;
    p->ucComponentsInScan = inf->p.ncomp_in_scan;
    p->ucHuffTableUsed = inf->p.huff_defined;
    p->iResInterval = inf->restart_interval;
}

static int init_common(JPEGIMAGE *p)
{
    JDInfo *inf = (JDInfo *)malloc(sizeof(JDInfo));
    if (!inf) { p->iError = JPEG_ERROR_MEMORY; return 0; }
    int rc = jd_parse_header(p->pFileData, p->iFileSize, 0, inf);
    /* fields the reference fills while it walks the markers, even when open fails later */
    fill_from_info(p, inf);
    p->ucOrientation = (uint8_t)inf->orientation;
    p->ucHasThumb = (uint8_t)inf->has_thumb;
    p->iThumbWidth = inf->thumb_w;
    p->iThumbHeight = inf->thumb_h;
    p->iThumbData = inf->thumb_data;
    p->iEXIF = inf->exif;
    p->iError = rc ? JPEG_SUCCESS : inf->error;
    p->parsed.scan_offset = inf->scan_offset;
    free(inf);
    p->pFramebuffer = NULL; /* must be set after open (jpeg.inl:1580) */
    return rc;
}

int JPEG_openRAM(JPEGIMAGE *p, uint8_t *pData, int iDataSize, JPEG_DRAW_CALLBACK *pfnDraw)
{
    memset(p, 0, sizeof(JPEGIMAGE));
    p->ucMemType = JPEG_MEM_RAM;
    p->pfnDraw = pfnDraw;
    p->JPEGFile.iSize = iDataSize;
    p->JPEGFile.pData = pData;
    p->iMaxMCUs = 1000;
    p->iDevice = -1;
    p->pFileData = pData;
    p->iFileSize = iDataSize;
    if (!pData || iDataSize <= 0) { p->iError = JPEG_INVALID_FILE; return 0; }
    return init_common(p);
}

/* whole file through the user's (or stdio) callbacks */
static int slurp(JPEGIMAGE *p)
{
    int size = p->JPEGFile.iSize;
    if (size <= 0) { p->iError = JPEG_INVALID_FILE; return 0; }
    uint8_t *buf = (uint8_t *)malloc((size_t)size + 16);
    if (!buf) { p->iError = JPEG_ERROR_MEMORY; return 0; }
    int got = 0;
    if (p->pfnSeek) (*p->pfnSeek)(&p->JPEGFile, 0);
    while (got < size) {
        int want = size - got; if (want > 65536) want = 65536;
        int r = (*p->pfnRead)(&p->JPEGFile, buf + got, want);
        if (r <= 0) break;
        got += r;
    }
    memset(buf + got, 0, (size_t)(size - got) + 16);
    p->pFileData = buf;
    p->iFileSize = got;
    p->bOwnsFileData = 1;
    return 1;
}

static int32_t file_read(JPEGFILE *f, uint8_t *buf, int32_t len)
{
    if (len > f->iSize - f->iPos) len = f->iSize - f->iPos;
    if (len <= 0) return 0;
    int32_t r = (int32_t)fread(buf, 1, (size_t)len, (FILE *)f->fHandle);
    f->iPos += r;
    return r;
}
static int32_t file_seek(JPEGFILE *f, int32_t pos)
{
    if (pos < 0) pos = 0; else if (pos >= f->iSize) pos = f->iSize - 1;
    f->iPos = pos;
    fseek((FILE *)f->fHandle, pos, SEEK_SET);
    return pos;
}
static void file_close(void *h) { if (h) fclose((FILE *)h); }

int JPEG_openFile(JPEGIMAGE *p, const char *szFilename, JPEG_DRAW_CALLBACK *pfnDraw)
{
    memset(p, 0, sizeof(JPEGIMAGE));
    p->ucMemType = JPEG_MEM_RAM;
    p->pfnRead = file_read;
    p->pfnSeek = file_seek;
    p->pfnDraw = pfnDraw;
    p->pfnClose = file_close;
    p->iMaxMCUs = 1000;
    p->iDevice = -1;
    FILE *f = fopen(szFilename, "rb");
    if (!f) return 0;
    p->JPEGFile.fHandle = f;
    fseek(f, 0, SEEK_END);
    p->JPEGFile.iSize = (int32_t)ftell(f);
    fseek(f, 0, SEEK_SET);
    if (!slurp(p)) return 0;
    return init_common(p);
}

int JPEG_openCallbacks(JPEGIMAGE *p, const char *szFilename, void *fHandle, int iDataSize, JPEG_OPEN_CALLBACK *pfnOpen,
                       JPEG_CLOSE_CALLBACK *pfnClose, JPEG_READ_CALLBACK *pfnRead, JPEG_SEEK_CALLBACK *pfnSeek,
                       JPEG_DRAW_CALLBACK *pfnDraw)
{
    memset(p, 0, sizeof(JPEGIMAGE));
    p->pfnRead = pfnRead; p->pfnSeek = pfnSeek; p->pfnDraw = pfnDraw; p->pfnOpen = pfnOpen; p->pfnClose = pfnClose;
    p->iMaxMCUs = 1000;
    p->iDevice = -1;
    if (!pfnRead) { p->iError = JPEG_INVALID_PARAMETER; return 0; }
    if (pfnOpen) {
        int32_t sz = 0;
        p->JPEGFile.fHandle = (*pfnOpen)(szFilename, &sz);
        p->JPEGFile.iSize = sz;
        if (p->JPEGFile.fHandle == NULL) return 0;
    } else {
        p->JPEGFile.fHandle = fHandle;
        p->JPEGFile.iSize = iDataSize;
    }
    if (!slurp(p)) return 0;
    return init_common(p);
}

void JPEG_close(JPEGIMAGE *p)
{
    if (p->pfnClose) (*p->pfnClose)(p->JPEGFile.fHandle);
    if (p->bOwnsFileData && p->pFileData) free(p->pFileData);
    p->pFileData = NULL;
    p->bOwnsFileData = 0;
    p->pfnClose = NULL;
}

int JPEG_getLastError(JPEGIMAGE *p) { return p->iError; }
int JPEG_getWidth(JPEGIMAGE *p) { return p->iWidth; }
int JPEG_getHeight(JPEGIMAGE *p) { return p->iHeight; }
int JPEG_getOrientation(JPEGIMAGE *p) { return (int)p->ucOrientation; }
int JPEG_getBpp(JPEGIMAGE *p) { return (int)p->ucBpp; }
int JPEG_getSubSample(JPEGIMAGE *p) { return (int)p->ucSubSample; }
int JPEG_getJPEGType(JPEGIMAGE *p) { return (p->ucMode == 0xc2) ? JPEG_MODE_PROGRESSIVE : JPEG_MODE_BASELINE; }
int JPEG_hasThumb(JPEGIMAGE *p) { return (int)p->ucHasThumb; }
int JPEG_getThumbWidth(JPEGIMAGE *p) { return p->iThumbWidth; }
int JPEG_getThumbHeight(JPEGIMAGE *p) { return p->iThumbHeight; }
void JPEG_setPixelType(JPEGIMAGE *p, int iType) { p->ucPixelType = (uint8_t)iType; }
int JPEG_getPixelType(JPEGIMAGE *p) { return (int)p->ucPixelType; }
void JPEG_setMaxOutputSize(JPEGIMAGE *p, int iMaxMCUs) { if (iMaxMCUs < 1) iMaxMCUs = 1; p->iMaxMCUs = iMaxMCUs; }
void JPEG_setUserPointer(JPEGIMAGE *p, void *u) { p->pUser = u; }
void JPEG_setFramebuffer(JPEGIMAGE *p, void *fb) { p->pFramebuffer = fb; }
void JPEG_setArithMode(JPEGIMAGE *p, int iMode) { p->ucArithMode = (uint8_t)(iMode ? JPEG_ARITH_SCALAR : JPEG_ARITH_SSE2); }
void JPEG_setDevice(JPEGIMAGE *p, int iDevice) { p->iDevice = iDevice; }
int JPEG_sizeofImage(void) { return (int)sizeof(JPEGIMAGE); }

static void mcu_size(int subsample, int *w, int *h)
{
    switch (subsample) {
        case 0x12: *w = 8; *h = 16; break;
        case 0x21: *w = 16; *h = 8; break;
        case 0x22: *w = 16; *h = 16; break;
        default: *w = 8; *h = 8; break;
    }
}

/* snap the crop to MCU boundaries, grow to cover the request (semantics of jpeg.inl:682-727) */
void JPEG_setCropArea(JPEGIMAGE *p, int x, int y, int w, int h)
{
    int mw, mh;
    mcu_size(p->ucSubSample, &mw, &mh);
    if (x < 0) x = 0;
    if (y < 0) y = 0;
    w = (w + mw - 1) / mw * mw;
    h = (h + mh - 1) / mh * mh;
    if (x > p->iWidth - mw) x = p->iWidth - mw;
    if (y > p->iHeight - mh) y = p->iHeight - mh;
    if (x + w > p->iWidth) w = p->iWidth - mw;
    if (y + h > p->iHeight) h = p->iHeight - mh;
    x &= ~(mw - 1);
    y &= ~(mh - 1);
    p->iCropX = x; p->iCropY = y; p->iCropCX = w; p->iCropCY = h;
}

void JPEG_getCropArea(JPEGIMAGE *p, int *x, int *y, int *w, int *h)
{
    *x = p->iCropX; *y = p->iCropY; *w = p->iCropCX; *h = p->iCropCY;
}

/* ---- decode ---- */
static int bits_per_pixel(int pt)
{
    switch (pt) {
        case RGB8888: return 32;
        case EIGHT_BIT_GRAYSCALE: return 8;
        case FOUR_BIT_DITHERED: return 4;
        case TWO_BIT_DITHERED: return 2;
        case ONE_BIT_DITHERED: return 1;
        default: return 16;
    }
}

/* ------------------------------------------------------------------------------------------------------------------
 * Delivery.  The GPU decodes the whole MCU-aligned frame; what remains of DecodeJPEG (src/jpeg.inl:5008-5127, :5300-5336)
 * is WHICH pixels go WHERE.  That is pure geometry, so it is computed first, as a list of draw items, and only then
 * executed: a draw item = a run of consecutive MCUs of one MCU row that the reference hands to the callback in one call.
 * The reference's rules (kept, quirks included, because callers see them):
 *   - MCU column x of row y is skipped when the row starts above the crop (y * mcuH < cropY) or when x * mcuW lies outside
 *     [cropX, cropX + cropW] -- both ends inclusive, so one MCU past the crop's right edge is still delivered (:5111, :5135);
 *   - a group is flushed when it is full or when the row's last MCU column has just been placed (:5300); a row whose last
 *     column is skipped never flushes a partial group;
 *   - after a flush the next group's width shrinks to what is left of the crop or of the row, rounded up to whole MCUs
 *     (:5327-5335); the width the callback may use is trimmed at the scaled image's right edge, else at the crop (:5313-5317);
 *   - with crop x scale the tests above compare SCALED MCU positions with the unscaled crop rectangle (SURVEY.md A.5): the
 *     outcome (e.g. no callbacks at all at 1/4 and 1/8) is reproduced literally.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
    int width, height;                  /* image size (full scale) */
    int crop_x, crop_y, crop_w, crop_h;
    int x_off, y_off;                   /* JPEG_decode placement */
    int subsample, pixel_type, options, max_mcus;
} JDDeliveryGeom;

typedef struct {
    int32_t mcu_row, mcu_col0, n_mcus;  /* the MCUs this call carries: n_mcus consecutive columns from mcu_col0 */
    int32_t x, y, w, h, w_used;         /* JPEGDRAW fields (w = iWidth = pitch of the block group in pixels) */
    int32_t buf;                        /* JPEG_USES_DMA: which half of the pixel buffer (0 / 1) */
} JDDrawItem;

static int scale_shift_of(int options)
{
    return (options & JPEG_SCALE_HALF) ? 1 : (options & JPEG_SCALE_QUARTER) ? 2 : (options & JPEG_SCALE_EIGHTH) ? 3 : 0;
}

/* Fills items[] (at most cap) and returns the number of draw calls the reference makes for this geometry; exported for
 * the CPU test tier, which compares it with the reference's own callback log (no GPU needed). */
int jd_delivery_schedule(const JDDeliveryGeom *g, JDDrawItem *items, int cap)
{
    const int shift = scale_shift_of(g->options);
    int mw, mh;
    mcu_size(g->subsample, &mw, &mh);
    const int cols = (g->width + mw - 1) / mw;
    const int rows = (g->crop_y + g->crop_h + mh - 1) / mh;      /* unscaled MCU height (:5014-5037) */
    mw >>= shift; mh >>= shift;
    const int pt = g->pixel_type;
    /* MCUs per draw call (:5062-5084) */
    int group = MAX_BUFFERED_PIXELS / (mw * mh);
    if (pt == RGB8888) group /= 2;
    if (pt == EIGHT_BIT_GRAYSCALE) group *= 2;
    if (group > cols) group = cols;
    int halves = 0;
    if (group > g->max_mcus) group = g->max_mcus;
    else if (g->options & JPEG_USES_DMA) { group /= 2; halves = 1; }
    if (pt > EIGHT_BIT_GRAYSCALE) group = cols;
    if (g->crop_w != g->width && group * mw > g->crop_w) group = g->crop_w / mw;
    if (group < 1) group = 1;
    const int round = (1 << shift) - 1;
    const int out_w = (g->width + round) >> shift, out_h = (g->height + round) >> shift;
    int n = 0, buf = 0;
    int h = mh;                                                   /* once trimmed it stays trimmed (jd.iHeight is never reset) */
    for (int r = 0; r < rows; r++) {
        const int row_above_crop = (r * mh < g->crop_y);
        int pitch = group * mw, filled = 0, first = -1;
        int x_px = g->x_off;
        for (int c = 0; c < cols; c++) {
            const int skip = row_above_crop || c * mw < g->crop_x || c * mw > g->crop_x + g->crop_w;
            if (skip) continue;
            if (filled == 0) first = c;
            filled += mw;
            if (filled != pitch && c != cols - 1) continue;
            /* flush */
            JDDrawItem it;
            it.mcu_row = r; it.mcu_col0 = first; it.n_mcus = filled / mw;
            it.x = x_px; it.w = it.w_used = pitch;
            if ((x_px - g->x_off) + pitch > out_w) it.w_used = out_w - (x_px - g->x_off);
            else if ((x_px - g->x_off) + pitch > g->crop_w) it.w_used = g->crop_w - (x_px - g->x_off);
            it.y = g->y_off + r * mh - g->crop_y;
            if ((it.y - g->y_off + mh) > out_h) h = out_h - (it.y - g->y_off);
            it.h = h;
            it.buf = buf;
            if (n < cap) items[n] = it;
            n++;
            if (halves) buf ^= 1;
            x_px += pitch;
            if (g->crop_w != cols * mw && (pitch + x_px) > (g->crop_x + g->crop_w)) pitch = g->crop_w - (x_px - g->x_off);
            else if ((cols - 1 - c) < group) pitch = (cols - 1 - c) * mw;
            if (pitch & (mw - 1)) pitch = (pitch + (mw - 1)) & ~(mw - 1);
            if (pitch < 0) pitch = 0;
            filled = 0;
        }
    }
    return n;
}

static void geom_of(const JPEGIMAGE *p, JDDeliveryGeom *g)
{
    g->width = p->iWidth; g->height = p->iHeight;
    g->crop_x = p->iCropX; g->crop_y = p->iCropY; g->crop_w = p->iCropCX; g->crop_h = p->iCropCY;
    g->x_off = p->iXOffset; g->y_off = p->iYOffset;
    g->subsample = p->ucSubSample; g->pixel_type = p->ucPixelType; g->options = p->iOptions; g->max_mcus = p->iMaxMCUs;
}

/* framebuffer mode (:5114-5124): every non-skipped MCU goes to (x_mcu - first kept column, y - cropY) of a frame whose pitch
 * is the crop width; no callback */
static void deliver_framebuffer(const JPEGIMAGE *p, const uint8_t *frame, int frame_pitch, int bypp, int last_mcu)
{
    const int shift = scale_shift_of(p->iOptions);
    int mw, mh;
    mcu_size(p->ucSubSample, &mw, &mh);
    const int cols = (p->iWidth + mw - 1) / mw;
    const int rows = (p->iCropY + p->iCropCY + mh - 1) / mh;
    mw >>= shift; mh >>= shift;
    const int out_h = (p->iHeight + (1 << shift) - 1) >> shift;
    const int pitch_px = p->iCropCX;
    const int pt = p->ucPixelType;
    /* the reference's SSE2 colour paths store whole MCUs with no edge clipping (jpeg.inl:3409, :4006): the right-edge MCU runs
     * on into the start of the next line (and is partly overwritten later, in MCU order), the bottom MCU row continues below
     * the image -- which is why the caller's buffer must cover whole MCU rows (c_cmdline/main.c:180).  Same writes, same
     * order; clipped only at the end of that MCU-row-aligned buffer.  Every other path clips at the image edges
     * (:3520-3524, :4311-4332). */
    const int whole_mcus = p->ucArithMode == JPEG_ARITH_SSE2 && shift == 0 && p->ucNumComponents == 3 && pt <= RGB8888 &&
                           (p->ucSubSample == 0x11 || p->ucSubSample == 0x22);
    const size_t fb_px = (size_t)pitch_px * (size_t)(rows * mh - p->iCropY);
    for (int r = 0; r < rows; r++) {
        if (r * mh < p->iCropY) continue;
        const int ty = r * mh - p->iCropY;
        int xoff = 0;
        for (int c = 0; c < cols; c++) {
            if (last_mcu >= 0 && r * cols + c > last_mcu) return;       /* decode error: the loops stop after the failing MCU (:5128) */
            if (c * mw < p->iCropX || c * mw > p->iCropX + p->iCropCX) continue;
            /* The inclusive test above lets one MCU past the crop's right edge through (:5111).  In a framebuffer that MCU lies
             * beyond the pitch: most of the reference's pixel paths store it anyway, so it runs on into the next line and
             * clobbers the first pixels there (SURVEY.md A.4: 2 640 wrong pixels on tulips); some clip it
             * (JPEGPutMCU8BitGray 4:2:0, :3019).  It is never stored here: the framebuffer receives the cropped image the
             * callbacks deliver (documented deviation). */
            if (xoff >= pitch_px) continue;
            const uint8_t *src = frame + (size_t)r * mh * frame_pitch + (size_t)c * mw * bypp;
            if (whole_mcus) {
                for (int l = 0; l < mh; l++) {
                    const size_t at = (size_t)(ty + l) * pitch_px + xoff;
                    size_t n = (size_t)mw;
                    if (at >= fb_px) break;
                    if (at + n > fb_px) n = fb_px - at;
                    memcpy((uint8_t *)p->pFramebuffer + at * bypp, src + (size_t)l * frame_pitch, n * bypp);
                }
            } else {
                int lines = mh, px = pitch_px - xoff;
                if (r * mh + lines > out_h) lines = out_h - r * mh;
                if (px > mw) px = mw;
                for (int l = 0; l < lines; l++) {
                    const size_t at = (size_t)(ty + l) * pitch_px + xoff;
                    size_t n = (size_t)px;
                    if (at >= fb_px) break;
                    if (at + n > fb_px) n = fb_px - at;
                    memcpy((uint8_t *)p->pFramebuffer + at * bypp, src + (size_t)l * frame_pitch, n * bypp);
                }
            }
            xoff += mw;
        }
    }
}

static int decode_common(JPEGIMAGE *p)
{
    int options = p->iOptions;
    if (!p->pFileData) { p->iError = JPEG_INVALID_PARAMETER; return 0; }
    /* progressive: DC-only 1/8 image (jpeg.inl:4964-4966), unless decoded from all scans (JPEGB200_OPT_PROGRESSIVE) */
    if (p->ucMode == 0xc2 && !(options & JPEGB200_OPT_PROGRESSIVE)) options = (p->iOptions |= JPEG_SCALE_EIGHTH);
    if (options & JPEG_EXIF_THUMBNAIL) {
        if (p->iThumbData == 0 || p->iThumbWidth == 0) { p->iError = JPEG_INVALID_PARAMETER; return 0; } /* jpeg.inl:4969 */
    }
    const int shift = scale_shift_of(options);
    if ((options & JPEG_LUMA_ONLY) && p->ucPixelType < EIGHT_BIT_GRAYSCALE) p->ucPixelType = EIGHT_BIT_GRAYSCALE; /* :4991 */
    if (p->ucPixelType >= INVALID_PIXEL_TYPE) { p->iError = JPEG_INVALID_PARAMETER; return 0; }
    const int pt = p->ucPixelType;
    const int dither = pt > EIGHT_BIT_GRAYSCALE;
    if (dither && !p->pDitherBuffer) { p->iError = JPEG_INVALID_PARAMETER; return 0; }
    if (!p->pFramebuffer && !p->pfnDraw) { p->iError = JPEG_INVALID_PARAMETER; return 0; }

    /* ---- the GPU part: whole MCU-aligned frame into a pinned staging buffer (holds the context's lock only) ---- */
    pthread_mutex_t *ctx_lock = NULL;
    JPEGB200_CTX *ctx = get_ctx(p->iDevice, p->ucArithMode, &ctx_lock);
    if (!ctx) { p->iError = JPEG_ERROR_MEMORY; return 0; }
    pthread_mutex_lock(ctx_lock);
    const uint8_t *datas[1] = {p->pFileData};
    int32_t sizes[1] = {p->iFileSize};
    JPEGB200_BATCH *b = JPEGB200_batchCreate(ctx, datas, sizes, 1, pt, (options & (0xFF | JPEGB200_OPT_PROGRESSIVE)) | JPEGB200_OPT_PADDED);
    if (!b) { pthread_mutex_unlock(ctx_lock); p->iError = JPEG_ERROR_MEMORY; return 0; }
    int32_t w = 0, h = 0, sub = 0, fw = 0, fh = 0, st = 0;
    JPEGB200_batchImageInfo(b, 0, &w, &h, &sub, &fw, &fh, &st);
    if (st != JPEG_SUCCESS) { JPEGB200_batchDestroy(b); pthread_mutex_unlock(ctx_lock); p->iError = st; return 0; }
    if (options & JPEG_EXIF_THUMBNAIL) { /* the reference re-parses into the same state (:4975) */
        p->iWidth = p->iCropCX = w; p->iHeight = p->iCropCY = h; p->iCropX = p->iCropY = 0; p->ucSubSample = (uint8_t)sub;
    }
    int64_t fpitch = 0;
    const int64_t fbytes = JPEGB200_batchOutputBytes(b, 0, &fpitch);
    size_t stage_bytes = 0;
    uint8_t *stage = stage_get((size_t)fbytes + 64, &stage_bytes);
    if (!stage) { JPEGB200_batchDestroy(b); pthread_mutex_unlock(ctx_lock); p->iError = JPEG_ERROR_MEMORY; return 0; }
    JPEGB200_batchSetOutput(b, 0, stage, 0);
    int32_t dst_status = 0;
    const int ok = JPEGB200_batchUpload(b) && JPEGB200_batchDecode(b, 0) && JPEGB200_batchDownload(b);
    const int wrc = ok ? JPEGB200_batchWait(b, &dst_status) : 0;
    const int err_mcu = wrc ? JPEGB200_batchErrMcu(b, 0) : -1;
    JPEGB200_batchDestroy(b);
    pthread_mutex_unlock(ctx_lock);
    if (!wrc) { stage_put(stage, stage_bytes); p->iError = JPEG_ERROR_MEMORY; return 0; }
    int decode_failed = (dst_status != JPEG_SUCCESS);
    int last_mcu = (decode_failed && err_mcu >= 0) ? err_mcu : -1;   /* MCUs after the failing one are never delivered */
    {   /* a crop that reaches below the image (JPEG_setCropArea does not prevent it for small images) makes the reference walk
         * MCU rows that do not exist: it runs out of data and fails with JPEG_DECODE_ERROR after the real rows were delivered */
        int fmw, fmh;
        mcu_size(p->ucSubSample, &fmw, &fmh);
        const int cols0 = (p->iWidth + fmw - 1) / fmw, rows0 = (p->iHeight + fmh - 1) / fmh;
        if ((p->iCropY + p->iCropCY + fmh - 1) / fmh > rows0) {
            decode_failed = 1;
            if (last_mcu < 0 || last_mcu > rows0 * cols0 - 1) last_mcu = rows0 * cols0 - 1;
        }
    }

    /* ---- delivery (no lock held: the callback may call back into the library) ---- */
    int mw, mh;
    mcu_size(p->ucSubSample, &mw, &mh);
    const int cols = (p->iWidth + mw - 1) / mw;
    mw >>= shift; mh >>= shift;
    const int bpp = bits_per_pixel(pt);
    const int bypp = bpp >= 8 ? bpp / 8 : 1;
    const int frame_pitch = (int)fpitch;
    if (p->pFramebuffer) {
        deliver_framebuffer(p, stage, frame_pitch, bypp, last_mcu);
    } else {
        JDDeliveryGeom g;
        geom_of(p, &g);
        const int n_items = jd_delivery_schedule(&g, NULL, 0);
        JDDrawItem *items = (JDDrawItem *)malloc(sizeof(JDDrawItem) * (size_t)(n_items > 0 ? n_items : 1));
        if (!items) { stage_put(stage, stage_bytes); p->iError = JPEG_ERROR_MEMORY; return 0; }
        jd_delivery_schedule(&g, items, n_items);
        /* the pixel block the callback sees: same size as the reference's usPixels (2048 px + slack), 16-byte aligned; with
         * JPEG_USES_DMA the two halves alternate (:5073-5076, :5326) */
        uint16_t pixbuf_raw[MAX_BUFFERED_PIXELS + 64];
        uint16_t *pixbuf = (uint16_t *)(((uintptr_t)pixbuf_raw + 15) & ~(uintptr_t)15);
        /* a group that ends at the image's right edge before it is full (crop x scale) leaves the rest of the block unwritten:
         * stale bytes in the reference, zeros here */
        memset(pixbuf_raw, 0, sizeof(pixbuf_raw));
        const int dpitch = dither ? (cols * mw * bpp + 7) / 8 : 0;
        JPEGDRAW jd;
        memset(&jd, 0, sizeof(jd));
        jd.iBpp = bpp;
        jd.pUser = p->pUser;
        for (int i = 0; i < n_items; i++) {
            const JDDrawItem *it = &items[i];
            /* a decode error ends the MCU loops after the failing MCU (:5128): a group is delivered only if its last MCU was reached */
            if (last_mcu >= 0 && it->mcu_row * cols + it->mcu_col0 + it->n_mcus - 1 > last_mcu) break;
            if (dither) {
                /* packed rows come from the dither kernel: one whole MCU row per call, in the caller's dither buffer */
                memcpy(p->pDitherBuffer, stage + (size_t)it->mcu_row * mh * frame_pitch, (size_t)dpitch * mh);
                jd.pPixels = (uint16_t *)p->pDitherBuffer;
            } else {
                uint8_t *dst = (uint8_t *)(pixbuf + (it->buf ? MAX_BUFFERED_PIXELS / 2 : 0));
                const uint8_t *src = stage + (size_t)it->mcu_row * mh * frame_pitch + (size_t)it->mcu_col0 * mw * bypp;
                int px = it->n_mcus * mw;
                if (px > it->w) px = it->w;
                for (int l = 0; l < mh && px > 0; l++) memcpy(dst + (size_t)l * it->w * bypp, src + (size_t)l * frame_pitch, (size_t)px * bypp);
                jd.pPixels = (uint16_t *)dst;
            }
            jd.x = it->x; jd.y = it->y; jd.iWidth = it->w; jd.iWidthUsed = it->w_used; jd.iHeight = it->h;
            if (!(*p->pfnDraw)(&jd)) break;
        }
        free(items);
    }
    stage_put(stage, stage_bytes);
    if (decode_failed) { p->iError = JPEG_DECODE_ERROR; return 0; }
    return 1;
}

int JPEG_decode(JPEGIMAGE *p, int x, int y, int iOptions)
{
    p->iXOffset = x;
    p->iYOffset = y;
    p->iOptions = iOptions;
    return decode_common(p);
}

int JPEG_decodeDither(JPEGIMAGE *p, uint8_t *pDither, int iOptions)
{
    p->iOptions = iOptions;
    p->pDitherBuffer = pDither;
    return decode_common(p);
}
