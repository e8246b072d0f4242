/*
 * jd_device.cu -- batch decode pipeline on one H100: buffers, uploads, kernel launches,
 * CUDA-event stage timings, downloads.  Exposes the JPEGB200_* C ABI (include/jpegdec_b200.h).
 * There is no CPU fallback anywhere in this file: if CUDA is unavailable every entry point fails.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <algorithm>
#include <unordered_map>
#include <time.h>
#include <new>
#include <sched.h>
#include <unistd.h>
#include <sys/syscall.h>

#include "jd_kernels.cuh"

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            snprintf(ctx_err(), 256, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            return 0;                                                                              \
        }                                                                                          \
    } while (0)

/* error text of the calling thread (two host threads driving two contexts never share it) */
static thread_local char g_err[256];

/* Device allocations are recycled through the context: a decode job borrows buffers and hands them
 * back on destroy, so steady-state batches do no cudaMalloc/cudaFree (both synchronise the device). */
struct JDPool {
    struct Slot { void *p; size_t bytes; };
    std::vector<Slot> free_;
    cudaError_t get(size_t bytes, void **out, size_t *got)
    {
        int best = -1;
        for (size_t i = 0; i < free_.size(); i++)
            if (free_[i].bytes >= bytes && free_[i].bytes <= 2 * bytes + (1u << 20) && (best < 0 || free_[i].bytes < free_[best].bytes)) best = (int)i;
        if (best >= 0) { *out = free_[best].p; *got = free_[best].bytes; free_.erase(free_.begin() + best); return cudaSuccess; }
        cudaError_t e = cudaMalloc(out, bytes);
        if (e != cudaSuccess) { /* give cached memory back to the driver and retry once */
            cudaGetLastError();
            drain();
            e = cudaMalloc(out, bytes);
        }
        *got = bytes;
        return e;
    }
    void put(void *p, size_t bytes) { free_.push_back(Slot{p, bytes}); }
    void drain() { for (auto &s : free_) cudaFree(s.p); free_.clear(); }
};

/* Pinned host staging blocks (status read-back) recycled the same way: a D2H copy into pageable memory would make
 * batchDownload wait for the whole job, which is what keeps several jobs from being in flight from one host thread. */
struct JDPinPool {
    struct Slot { void *p; size_t bytes; };
    std::vector<Slot> free_;
    void *get(size_t bytes, size_t *got)
    {
        for (size_t i = 0; i < free_.size(); i++)
            if (free_[i].bytes >= bytes) { void *q = free_[i].p; *got = free_[i].bytes; free_.erase(free_.begin() + i); return q; }
        void *q = nullptr;
        size_t need = (bytes + 4095) & ~(size_t)4095;
        if (cudaHostAlloc(&q, need, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        *got = need;
        return q;
    }
    void put(void *p, size_t bytes) { free_.push_back(Slot{p, bytes}); }
    void drain() { for (auto &s : free_) cudaFreeHost(s.p); free_.clear(); }
};

/* a job's stream and its timing events, recycled through the context (creating them costs more than a small decode) */
struct JDStreamSet {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[JPEGB200_NUM_TIMINGS + 2] = {};
    bool complete() const { return stream && ev[JPEGB200_NUM_TIMINGS + 1]; }   /* created in this order */
    void destroy()
    {
        for (auto &e : ev) if (e) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
    }
};

struct JPEGB200_CTX {
    std::vector<JDStreamSet> free_streams;
    int device;
    int arith;
    bool has_shared;
    uint64_t shared_hash, shared_hash2;
    uint16_t shared_lut[JD_LUT_ENTRIES];
    int shared_hits;
    JDPool pool;
    JDPinPool pinpool;
    int64_t last_counters[JPEGB200_NUM_COUNTERS]; /* summed over the jobs of the last JPEGB200_decodeBatch */
    float last_ms[JPEGB200_NUM_TIMINGS];          /* CUDA-event stage times summed over those jobs */
    int last_jobs;
    int numa_node;                                /* host NUMA node the GPU hangs off (-1 unknown) */
    int pipe_depth;                               /* jobs in flight inside JPEGB200_decodeBatch (0 = default) */
};

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

/* A device buffer borrowed from a pool; it goes back when the buffer dies.  Movable, not copyable: a copy would hand the
 * same pointer to the pool twice. */
template <typename T>
struct DevBuf {
    T *p = nullptr;
    size_t n = 0;
    size_t bytes = 0;
    JDPool *pool = nullptr;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    DevBuf(DevBuf &&o) noexcept : p(o.p), n(o.n), bytes(o.bytes), pool(o.pool) { o.p = nullptr; o.n = 0; o.bytes = 0; }
    ~DevBuf() { release(); }
    cudaError_t alloc(JDPool *from, size_t count)
    {
        if (count <= n && p) return cudaSuccess;
        release();
        pool = from;
        size_t need = align256((count ? count : 1) * sizeof(T));
        void *q = nullptr;
        cudaError_t e = pool ? pool->get(need, &q, &bytes) : cudaMalloc(&q, bytes = need);
        if (e == cudaSuccess) { p = (T *)q; n = count; }
        return e;
    }
    void release()
    {
        if (p) { if (pool) pool->put(p, bytes); else cudaFree(p); }
        p = nullptr; n = 0; bytes = 0;
    }
};

/* One job.  Every member starts empty; the DevBuf members return to the context's pool when the batch is deleted
 * (JPEGB200_batchDestroy, after the stream has drained). */
struct JPEGB200_BATCH {
    JPEGB200_CTX *ctx = nullptr;
    int n = 0;                      /* images (views with JPEGB200_batchCreateViews): everything per image is per view */
    /* nf files, each walked once through its entropy-facing descriptor fdescs[f] (d_fdescs), where the kernels write its
     * status; descs[i] is view i's descriptor for the IDCT and after it, carrying its file's seg / blk / rec bases.
     * Without views every file has one view: n = nf and vfile[i] = i. */
    int nf = 0;
    std::vector<int32_t> vfile;     /* per view: its file */
    std::vector<JDImageDesc> fdescs;
    DevBuf<JDImageDesc> d_fdescs;
    int pixel_type = 0, options = 0, sshift = 0, ptclass = 0, dither_bits = 0;
    bool gray_out = false;
    bool padded = false; /* write the whole MCU-aligned frame (single-image API: callbacks deliver whole MCUs) */
    bool roi = false;    /* created with regions of interest or orientations (JPEGB200_batchCreateOriented) */
    std::vector<JDRoiPlan> plans;   /* per image, with roi */
    std::vector<int32_t> exif_tag;  /* per image: the file's EXIF Orientation tag (0 = none) */
    std::vector<uint8_t> orient;    /* per image: the transform applied, 1-8 (1 without orients) */
    uint32_t nseg_walk = 0;         /* restart intervals the entropy stage walks (JPEGB200_C_SEGMENTS) */
    /* resize (JPEGB200_batchCreateResized): descs hold the resized size; the IDCT stage writes S (the unresized output,
     * rs_src_w x rs_src_h) into d_rs, the resize passes write the destination */
    bool resize = false;
    int rs_filter = 0;
    std::vector<JDResizePlan> rs_plans;
    std::vector<uint32_t> rs_src_w, rs_src_h;
    std::vector<int64_t> rs_scratch;    /* per image: S + intermediate bytes in d_rs (256-byte aligned each) */
    int64_t rs_scratch_total = 0;
    std::vector<JDResizeDesc> rs_desc;
    DevBuf<uint8_t> d_rs;
    DevBuf<int32_t> d_rs_coef;
    DevBuf<JDResizeDesc> d_rs_desc;
    /* box resize (JPEGB200_batchCreateBox with boxes or gaps): every view resizes through its box plan; a reduce writes the
     * resize source after S in d_rs */
    bool box = false;
    std::vector<JDBoxPlan> bx_plans;
    std::vector<JDBoxDesc> bx_desc;
    DevBuf<JDBoxDesc> d_bx_desc;
    /* windows (JPEGB200_batchCreateWindow): every view resizes (to S's own size without out_sizes) into its window.  Per
     * view its plan, its window and the full S (before the decode is narrowed to the support) */
    bool window = false;
    std::vector<JDWindowPlan> wn_plans;
    std::vector<int32_t> wn_full;       /* 2 per view */
    std::vector<int32_t> wn_out;        /* 2 per view: R's size */
    std::vector<int32_t> wn_win;        /* 4 per view: the window */
    /* colour operations (JPEGB200_batchCreateColor): per view its plan and byte order; jdk_color rewrites the view's final
     * uint8 image in place, before jdk_tensor */
    bool color = false;
    std::vector<JDColorPlan> co_plans;
    std::vector<JDBlurPlan> co_blur;        /* per view: each blur's constants at its op slot */
    std::vector<JDAugPlan> co_aug;          /* per view: each geometric op's mapping at its op slot */
    std::vector<JDResamplePlan> co_rs;      /* per view: each BILINEAR / BICUBIC geometric op's matrix at its op slot */
    std::vector<JDWarpPlan> co_warp;        /* per view, for a batch created with warp arguments: each AFFINE / PERSPECTIVE
                                               op's coefficients and fill at its op slot */
    std::vector<int64_t> bl_scratch;        /* per view: its scratch copy's bytes when it blurs, sharpens or moves pixels
                                               (256-byte aligned), plus JD_AU_HIST counts per autocontrast / equalize */
    int64_t bl_scratch_total = 0;
    std::vector<JDBlurDesc> bl_desc;        /* per blur launch pair, per view blurring there */
    std::vector<uint32_t> bl_blk;           /* the same entries: first CTA of the horizontal, then of the vertical kernel */
    DevBuf<JDBlurDesc> d_bl_desc;
    DevBuf<uint32_t> d_bl_blk;
    DevBuf<uint8_t> d_bl;                   /* the scratch copies */
    std::vector<JDAugDesc> au_desc;         /* per cut index, per view sharpening or moving pixels there (jdk_augment, _rs, _copy) */
    DevBuf<JDAugDesc> d_au_desc;
    std::vector<JDAugMat> au_mat;           /* the same entries: the BILINEAR / BICUBIC ops' matrices (zero for the others) */
    DevBuf<JDAugMat> d_au_mat;
    std::vector<JDWarpDesc> au_warp;        /* the same entries: the AFFINE / PERSPECTIVE ops' coefficients and fill (zero for the others) */
    DevBuf<JDWarpDesc> d_au_warp;
    std::vector<int16_t> au_tab;            /* the walk tables of the NEAREST affines with b = d = 0 (jd_au_walk_table) */
    DevBuf<int16_t> d_au_tab;
    std::vector<JDJqDesc> jq_desc;          /* per cut index, per view compressing there (jdk_jq_fwd, jdk_jq_color) */
    DevBuf<JDJqDesc> d_jq_desc;
    std::vector<uint16_t> jq_tab;           /* the table pair of each distinct quality in the batch (jd_jq_tables) */
    DevBuf<uint16_t> d_jq_tab;
    DevBuf<uint32_t> d_co_hslot;            /* per cut index and view: its histogram slot (the slots follow the scratch copies in d_bl) */
    std::vector<uint8_t> co_bgr;
    std::vector<JDColorDesc> co_desc;
    std::vector<uint32_t> co_blk;           /* per launch, per view: its first CTA */
    DevBuf<JDColorDesc> d_co_desc;
    DevBuf<uint32_t> d_co_blk;
    DevBuf<unsigned long long> d_co_sum;    /* per view, per contrast: the sum of L before it */
    /* tensor output (JPEGB200_batchCreateTensor): descs hold the row bytes as out_pitch; the pipeline (IDCT or resize) writes
     * U (out_w x out_h, tn_bpp bytes per pixel) tightly into d_tn, jdk_tensor writes the destination */
    bool tensor = false;
    JPEGB200_TensorSpec tn_spec = {};
    int tn_elt = 0, tn_nc = 0, tn_bpp = 0, tn_planes = 0;   /* tn_planes: C for CHW (the tensor is tn_planes x out_h rows), 1 for HWC */
    std::vector<uint8_t> tn_swap;           /* per image: output channel c reads byte 2 - c of a staged pixel */
    std::vector<int64_t> tn_stage;          /* per image: staging bytes (256-byte aligned) */
    std::vector<int64_t> tn_plane;          /* per image: the caller's plane stride (0 = pitch * out_h) */
    int64_t tn_stage_total = 0;
    std::vector<uint32_t> tn_table;         /* 3 x 256 elements, zero-extended to 32 bits */
    std::vector<JDTensorDesc> tn_desc;
    DevBuf<uint8_t> d_tn;
    DevBuf<uint32_t> d_tn_tab;
    DevBuf<JDTensorDesc> d_tn_desc;
    JDStreamSet ss;                 /* from the context on first use (batch_stream), back to it on destroy */
    std::vector<JDInfo> infos;
    std::vector<int32_t> parse_status;
    std::vector<const uint8_t *> datas;
    std::vector<int32_t> sizes;
    std::vector<JDImageDesc> descs;
    std::vector<int32_t> quant;
    std::vector<uint16_t> luts;
    std::vector<uint32_t> work, cta_lut, seg_img;
    std::vector<uint64_t> comp_off; /* offset of each file in the device blob */
    std::vector<void *> outs;
    std::vector<int64_t> pitches;
    int index_base = 0;             /* index of image 0 in the caller's list (JPEGB200_decodeBatch jobs): error messages */
    std::vector<uint16_t> errinit;  /* dither: initial error line per image (reference quirk), value | 0xFF00 (tag of "the band above band 0") */
    size_t comp_total = 0, out_total = 0, gray_total = 0;
    uint32_t nseg = 0, nlut = 0;
    uint64_t nblk = 0;
    bool contiguous_in = false;
    bool uploaded = false, out_device = false, arena_owned = false;
    DevBuf<uint8_t> d_comp, d_out, d_gray;
    DevBuf<uint16_t> d_errline;
    DevBuf<uint64_t> d_gray_off; /* [0,n): gray-stage offsets, [n,2n): packed output offsets, [2n,3n): output pitches */
    DevBuf<uint32_t> d_err_off, d_dprog;
    DevBuf<uint8_t> d_clean;       /* un-stuffed restart segments (jdk_unstuff_segs) */
    DevBuf<uint32_t> d_seg_clen;
    uint64_t rec_total = 0;        /* coefficient records the batch may need (JD_REC_INDEX layout) */
    DevBuf<uint4> d_dbands;        /* dither: (image, band, list position of the band above, of band - 255 or ~0) per warp */
    std::vector<uint4> dbands;
    JDImageDesc *descs_dl = nullptr;   /* descriptors read back (status, err_mcu); pinned, from ctx->pinpool */
    size_t descs_dl_bytes = 0;
    bool downloaded = false;
    DevBuf<JDImageDesc> d_descs;
    DevBuf<int32_t> d_quant;
    DevBuf<uint16_t> d_luts, d_rec;
    DevBuf<uint32_t> d_work, d_cta_lut, d_seg_img, d_seg_start, d_seg_jmap, d_seg_status, d_seg_nrec, d_seg_phase, d_counters;
    DevBuf<jd_u64> d_blk_hdr;
    DevBuf<JDEvent> d_events;
    std::vector<uint64_t> arena_off; /* per-image offset inside d_out */
    /* restart-free scans decoded chunk-parallel (jd_chunk.h) */
    std::vector<uint32_t> cimg_list;
    uint32_t nchunks = 0, max_nch = 0;
    DevBuf<uint8_t> d_filt;
    DevBuf<uint32_t> d_cimg_list, d_flen, d_E0, d_E1, d_Ep, d_cfirst, d_cn, d_cpre, d_cjmap, d_cstatus, d_cnown;
    DevBuf<int32_t> d_cdcs, d_cpe;
    /* progressive files decoded from all their scans (JPEGB200_OPT_PROGRESSIVE, jd_prog.h) */
    std::vector<JDProgScan> pscans;      /* the walkers: by wave, longest scan first inside a wave */
    std::vector<uint32_t> pwave_off;     /* wave w: pscans[pwave_off[w] .. pwave_off[w + 1]) */
    std::vector<JDProgHuff> ptabs;       /* the batch's decoder tables, one per distinct content */
    std::vector<JDProgFile> pfiles;
    std::vector<int64_t> pplane;         /* per file: coefficient plane bytes (0: no such plane) */
    int64_t pplane_total = 0;
    uint32_t pwalkers = 0;               /* walkers of files whose plane was allocated (JPEGB200_C_SEGMENTS) */
    std::vector<DevBuf<int16_t>> d_pplane;
    std::vector<int16_t *> pplane_ptr;
    DevBuf<JDProgScan> d_pscans;
    DevBuf<JDProgHuff> d_ptabs;
    DevBuf<JDProgFile> d_pfiles;
    DevBuf<int16_t *> d_pplanes;
    DevBuf<uint32_t> d_perr;
    /* libjpeg's default decompression (JPEGB200_OPT_LIBJPEG, jd_ljpeg.h): per image its MCU box and planes */
    bool lj = false;
    std::vector<JDLjDesc> lj_desc;
    std::vector<int64_t> lj_plane;       /* per image: plane bytes (256-byte aligned; 0 for a failed image) */
    int64_t lj_plane_total = 0;
    uint32_t lj_max_blocks = 0, lj_max_pixels = 0;
    uint32_t lj_s_blocks[4] = {}, lj_s_pixels[4] = {};   /* the same per draft shift 1-3 (JPEGB200_batchCreateDraft) */
    DevBuf<uint8_t> d_lj;
    DevBuf<JDLjDesc> d_lj_desc;
    uint32_t h_changed = 0;
    bool chunk_iterate = false;  /* restart-free scans: iterate the entry states with a host check (fallback mode) */
    int decode_flags = 0;
    float ms[JPEGB200_NUM_TIMINGS] = {};
    int64_t counters[JPEGB200_NUM_COUNTERS] = {};
    uint32_t *h_counters = nullptr;    /* 8 words at the end of the descs_dl block */
};

static char *ctx_err() { return g_err; }

#define JD_EVENT_CAP (1u << 20)
#define JD_CHUNK_PASSES 6     /* restart-free scans: entry-state passes per decode (from the third on only moved chunks are parsed; the last one verifies) */

extern "C" int JPEGB200_deviceCount(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

/* the calling thread's current CUDA device (-1 without CUDA) */
extern "C" int JPEGB200_currentDevice(void)
{
    int d = -1;
    if (cudaGetDevice(&d) != cudaSuccess) { cudaGetLastError(); return -1; }
    return d;
}

extern "C" JPEGB200_CTX *JPEGB200_create(int device, int arith_mode)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        snprintf(g_err, sizeof(g_err), "no CUDA device: %s (this library has no CPU fallback)", cudaGetErrorString(e));
        return nullptr;
    }
    if (device < 0) { if (cudaGetDevice(&device) != cudaSuccess) device = 0; }
    if (device >= n) { snprintf(g_err, sizeof(g_err), "device %d out of range (%d devices)", device, n); return nullptr; }
    if (cudaSetDevice(device) != cudaSuccess) { snprintf(g_err, sizeof(g_err), "cudaSetDevice(%d) failed", device); return nullptr; }
    /* make sure the sm_90a kernel image is loadable on this GPU */
    cudaFuncAttributes fa;
    e = cudaFuncGetAttributes(&fa, jdk_prescan);
    if (e != cudaSuccess) {
        snprintf(g_err, sizeof(g_err), "kernel image not loadable on device %d: %s (built for sm_90a only)", device, cudaGetErrorString(e));
        cudaGetLastError();
        return nullptr;
    }
    JPEGB200_CTX *c = new (std::nothrow) JPEGB200_CTX();
    if (!c) return nullptr;
    c->device = device;
    c->arith = arith_mode ? JPEG_ARITH_SCALAR : JPEG_ARITH_SSE2;
    c->has_shared = false;
    c->shared_hits = 0;
    memset(c->last_counters, 0, sizeof(c->last_counters));
    memset(c->last_ms, 0, sizeof(c->last_ms));
    c->last_jobs = 0;
    c->pipe_depth = 0;
    c->numa_node = -1;
    {   /* which host NUMA node is this GPU attached to?  (/sys/bus/pci/devices/<domain:bus:dev.fn>/numa_node) */
        char bus[32] = {0}, path[96];
        if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) == cudaSuccess) {
            for (char *q = bus; *q; q++) if (*q >= 'A' && *q <= 'Z') *q = (char)(*q - 'A' + 'a');
            snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
            FILE *f = fopen(path, "r");
            if (f) { int node = -1; if (fscanf(f, "%d", &node) == 1) c->numa_node = node; fclose(f); }
        } else cudaGetLastError();
    }
    return c;
}

extern "C" void JPEGB200_destroy(JPEGB200_CTX *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    ctx->pool.drain();
    ctx->pinpool.drain();
    for (auto &ss : ctx->free_streams) ss.destroy();
    delete ctx;
}

extern "C" const char *JPEGB200_lastErrorString(JPEGB200_CTX *) { return g_err; }

extern "C" void *JPEGB200_hostAlloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}

extern "C" void JPEGB200_hostFree(void *p) { if (p) cudaFreeHost(p); }

/* ---- host placement: the pixels of a batch leave the GPU over PCIe into pinned host memory; on a two-socket box that
 * memory (and the thread that drives the copies) should sit on the socket the GPU hangs off, or every byte crosses the
 * inter-socket link as well.  Nothing here is required for correctness. ---- */
extern "C" int JPEGB200_numaNode(JPEGB200_CTX *ctx) { return ctx ? ctx->numa_node : -1; }

/* parse "0-3,8,10-11" */
static int jd_parse_cpulist(const char *txt, cpu_set_t *set)
{
    int n = 0;
    CPU_ZERO(set);
    const char *q = txt;
    while (*q) {
        char *e;
        long a = strtol(q, &e, 10);
        if (e == q) break;
        long b2 = a;
        if (*e == '-') { q = e + 1; b2 = strtol(q, &e, 10); }
        for (long c = a; c <= b2 && c < CPU_SETSIZE; c++) { CPU_SET((int)c, set); n++; }
        q = e;
        while (*q == ',' || *q == ' ' || *q == '\n') q++;
    }
    return n;
}

/* Pins the CALLING thread (and the threads it creates later) to the CPUs of the context's NUMA node -- intersected with
 * the CPUs the process may use -- and makes that node the preferred one for its allocations; pinned memory allocated
 * afterwards (JPEGB200_hostAlloc) lands there.  Returns the number of CPUs in the new mask, 0 if nothing was changed. */
extern "C" int JPEGB200_bindHostToDevice(JPEGB200_CTX *ctx)
{
    if (!ctx || ctx->numa_node < 0) return 0;
    char path[96], txt[4096];
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", ctx->numa_node);
    FILE *f = fopen(path, "r");
    if (!f) return 0;
    const size_t got = fread(txt, 1, sizeof(txt) - 1, f);
    fclose(f);
    txt[got] = 0;
    cpu_set_t node, cur, both;
    if (jd_parse_cpulist(txt, &node) == 0) return 0;
    if (sched_getaffinity(0, sizeof(cur), &cur) != 0) return 0;
    CPU_AND(&both, &node, &cur);
    const int n = CPU_COUNT(&both);
    if (n == 0) return 0;
    if (sched_setaffinity(0, sizeof(both), &both) != 0) return 0;
#ifdef SYS_set_mempolicy
    {   /* MPOL_PREFERRED = 1: fall back to other nodes rather than fail when the node is full */
        unsigned long mask[16] = {0};
        if (ctx->numa_node < (int)(8 * sizeof(mask))) {
            mask[ctx->numa_node / (8 * sizeof(unsigned long))] |= 1ul << (ctx->numa_node % (8 * sizeof(unsigned long)));
            (void)syscall(SYS_set_mempolicy, 1, mask, (unsigned long)(8 * sizeof(mask)));
        }
    }
#endif
    return n;
}

extern "C" void *JPEGB200_deviceAlloc(JPEGB200_CTX *ctx, size_t bytes)
{
    if (!ctx || cudaSetDevice(ctx->device) != cudaSuccess) return nullptr;
    void *p = nullptr;
    if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}

extern "C" void JPEGB200_deviceFree(JPEGB200_CTX *ctx, void *p)
{
    if (ctx) cudaSetDevice(ctx->device);
    if (p) cudaFree(p);
}

extern "C" int JPEGB200_deviceRead(JPEGB200_CTX *ctx, void *host_dst, const void *dev_src, size_t bytes)
{
    if (!ctx) return 0;
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpy(host_dst, dev_src, bytes, cudaMemcpyDeviceToHost));
    return 1;
}

/* ---- digests of device-resident pixels: lets a caller (bench / tests) verify a whole device-resident batch against
 * reference digests without moving the pixels to the host.  digest = sum over 8-byte words i of mix64(word ^ i * K)
 * mod 2^64 (mix64 = the splitmix64 finaliser); order independent, so it reduces in parallel. ---- */
/* digests of n device byte ranges (8-byte aligned starts); synchronous */
extern "C" int JPEGB200_digestDevice(JPEGB200_CTX *ctx, const void *const *dev_ptrs, const int64_t *lengths, int n, uint64_t *digests)
{
    if (!ctx || n <= 0 || !dev_ptrs || !lengths || !digests) return 0;
    for (int i = 0; i < n; i++) if (((uintptr_t)dev_ptrs[i] & 7u) || lengths[i] < 0) { snprintf(g_err, sizeof(g_err), "digest ranges must start 8-byte aligned"); return 0; }
    CK(cudaSetDevice(ctx->device));
    void *d = nullptr;
    const size_t pb = (size_t)n * 8;
    CK(cudaMalloc(&d, 3 * pb));
    uint8_t *dp = (uint8_t *)d;
    int ok = 1;
    if (cudaMemcpy(dp, dev_ptrs, pb, cudaMemcpyHostToDevice) != cudaSuccess || cudaMemcpy(dp + pb, lengths, pb, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemset(dp + 2 * pb, 0, pb) != cudaSuccess) ok = 0;
    if (ok) {
        for (int i0 = 0; i0 < n; i0 += 32768) {
            const int cnt = (n - i0 < 32768) ? n - i0 : 32768;
            jdk_digest<<<dim3(64, cnt), 256>>>((const uint8_t *const *)dp + i0, (const int64_t *)(dp + pb) + i0, (unsigned long long *)(dp + 2 * pb) + i0);
        }
        if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(digests, dp + 2 * pb, pb, cudaMemcpyDeviceToHost) != cudaSuccess) ok = 0;
    }
    if (!ok) snprintf(g_err, sizeof(g_err), "digest failed: %s", cudaGetErrorString(cudaGetLastError()));
    cudaFree(d);
    return ok;
}

extern "C" int JPEGB200_setPipelineDepth(JPEGB200_CTX *ctx, int jobs_in_flight)
{
    if (!ctx || jobs_in_flight < 0 || jobs_in_flight > 16) return 0;
    ctx->pipe_depth = jobs_in_flight;
    return 1;
}

/* ---- shared table blob ---- */
extern "C" int JPEGB200_exportTables(const uint8_t *jpeg, int size, uint8_t *blob)
{
    JDInfo *info = new JDInfo();
    int rc = jd_parse_header(jpeg, size, 0, info);
    if (rc) {
        const uint64_t h = jd_tables_hash(info), h2 = jd_tables_hash2(info);   /* 128-bit key of the DHT content */
        memcpy(blob, &h, 8);
        memcpy(blob + 8, &h2, 8);
        jd_build_lut(info, (uint16_t *)(blob + 16));
        jd_build_quant(info, (int16_t *)(blob + 16 + JD_LUT_ENTRIES * 2));
    }
    delete info;
    return rc;
}

extern "C" int JPEGB200_setSharedTables(JPEGB200_CTX *ctx, const uint8_t *blob)
{
    if (!ctx) return 0;
    memcpy(&ctx->shared_hash, blob, 8);
    memcpy(&ctx->shared_hash2, blob + 8, 8);
    memcpy(ctx->shared_lut, blob + 16, JD_LUT_ENTRIES * 2);
    ctx->has_shared = true;
    ctx->shared_hits = 0;
    return 1;
}

extern "C" int JPEGB200_sharedTableHits(JPEGB200_CTX *ctx) { return ctx ? ctx->shared_hits : 0; }

/* ---- batch ---- */
static int bytes_per_pixel_class(int ptclass) { return ptclass == JD_PT_565 ? 2 : (ptclass == JD_PT_8888 ? 4 : 1); }

extern "C" uint64_t jd_rec_extent(uint64_t size, uint32_t scan_offset, uint32_t nseg, uint32_t nch)
{
    /* restart segment s: JD_REC_INDEX(start, s) + JD_REC_CAP(end - start) <= 6 end + 128 s + 120, and end <= size */
    uint64_t e = (uint64_t)JD_REC_PER_BYTE * size + (uint64_t)JD_REC_SLOT_SLACK * (nseg ? nseg - 1u : 0u) + JD_REC_SLOT_SLACK - 8u;
    if (nch) {   /* the last chunk, c = nch - 1 at slot nseg + c: its start is past the data, but its capacity counts */
        const uint64_t off = (uint64_t)scan_offset + (uint64_t)JD_CHUNK_BYTES * (nch - 1u);
        const uint64_t c = ((JD_REC_PER_BYTE * off) & ~(uint64_t)7) + (uint64_t)JD_REC_SLOT_SLACK * (nseg + nch - 1u) +
                           JD_REC_PER_BYTE * JD_CHUNK_BYTES + JD_REC_SLOT_SLACK - 8u;
        if (c > e) e = c;
    }
    return e;
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreate(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes,
                                                int n, int pixel_type, int options)
{
    return JPEGB200_batchCreateROI(ctx, datas, sizes, n, pixel_type, options, nullptr);
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateROI(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes,
                                                   int n, int pixel_type, int options, const int32_t *rois)
{
    return JPEGB200_batchCreateOriented(ctx, datas, sizes, n, pixel_type, options, rois, nullptr);
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateOriented(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes,
                                                        int n, int pixel_type, int options, const int32_t *rois,
                                                        const uint8_t *orients)
{
    return JPEGB200_batchCreateResized(ctx, datas, sizes, n, pixel_type, options, rois, orients, nullptr, 0);
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateResized(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes,
                                                       int n, int pixel_type, int options, const int32_t *rois,
                                                       const uint8_t *orients, const int32_t *out_sizes, int filter)
{
    return JPEGB200_batchCreateTensor(ctx, datas, sizes, n, pixel_type, options, rois, orients, out_sizes, filter, nullptr);
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateTensor(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes,
                                                      int n, int pixel_type, int options, const int32_t *rois,
                                                      const uint8_t *orients, const int32_t *out_sizes, int filter,
                                                      const JPEGB200_TensorSpec *spec)
{
    return JPEGB200_batchCreateViews(ctx, datas, sizes, n, nullptr, pixel_type, options, rois, orients, out_sizes, filter, spec);
}

/* ---- JPEGB200_batchCreateViews, step by step.  CreatePlan lives on its stack: the caller's per-view arguments and what
 * one file's steps hand to the next file's. ---- */
struct CreatePlan {
    const uint8_t *const *datas = nullptr;
    const int32_t *sizes = nullptr, *rois = nullptr, *out_sizes = nullptr;
    const int32_t *views = nullptr;     /* per file: its view count (all ones for a call without views) */
    const uint8_t *orients = nullptr;
    const JPEGB200_TensorSpec *spec = nullptr;
    const uint8_t *draft = nullptr;     /* per view: draft scale denominator (JPEGB200_batchCreateDraft), NULL = 1 */
    const double *boxes = nullptr, *gaps = nullptr;   /* per view: resize box and reducing gap (JPEGB200_batchCreateBox) */
    const JPEGB200_ColorOp *color = nullptr;          /* per view: JPEGB200_COLOR_MAX_OPS operations (JPEGB200_batchCreateColor) */
    const JPEGB200_WarpArgs *warp = nullptr;          /* per view: their AFFINE / PERSPECTIVE arguments (JPEGB200_batchCreateWarp) */
    const int32_t *windows = nullptr;                 /* per view: x, y, w, h (JPEGB200_batchCreateWindow) */
    /* with windows: the rectangles the views decode (the caller's rois narrowed to each window's support; rois points here)
     * and without out_sizes the resize targets (S's own size; out_sizes points here) */
    std::vector<int32_t> wn_rois, wn_sizes;
    const int32_t *caller_rois = nullptr;
    /* where the next file's restart segments, blocks and records start; where the next view's output and gray stage start */
    uint32_t seg = 0;
    uint64_t blk = 0, rec_total = 0;
    size_t out_total = 0, gray_total = 0;
    std::vector<uint64_t> lut_hash;
    std::vector<int> lut_owner;         /* first file that defined each LUT set: a hash match is confirmed on the DHT bytes */
    std::vector<int32_t> srects, vok;   /* per view: its rectangle in the stored frame (jd_views_plan), and whether it is valid */
    std::vector<uint8_t> ks;            /* per view, with orients: the transform asked for (above 8: refused by jd_views_plan) */
    std::vector<JDProgScan> fscans;     /* jd_prog_parse's scans and tables of the current file */
    std::vector<JDProgHuff> ftabs;
    std::unordered_map<uint64_t, std::vector<uint32_t>> ptab_index;   /* table content hash -> its indices in b->ptabs */
};

/* what admit_file and size_file_walk find out about one file */
struct FileAdmit {
    int ok = 0, status = JPEG_SUCCESS;
    bool prog = false, full = false;   /* prog: DC-only 1/8 decode of a progressive file; full: decoded from all its scans (jd_prog.h) */
    int nsc = 0, ntb = 0;              /* full: its scans and tables in CreatePlan::fscans / ftabs */
    uint32_t total_mcus = 0, mps = 0, nseg = 0, nch = 0;
};

/* the batch's fixed state from the (checked) arguments: feature flags, pixel class, per-view and per-file vectors sized */
static void init_batch(JPEGB200_BATCH *b, JPEGB200_CTX *ctx, const CreatePlan &P, int n, int nv, int pixel_type, int options, int filter)
{
    b->ctx = ctx;
    b->n = nv;
    b->nf = n;
    b->roi = P.rois != nullptr || P.orients != nullptr;
    b->plans.assign(nv, JDRoiPlan{});   /* read with rois or orients only */
    b->exif_tag.assign(nv, 0);
    b->orient.assign(nv, 1);
    pixel_type = jd_fold_luma_only(pixel_type, options);
    b->pixel_type = pixel_type;
    b->padded = (options & JPEGB200_OPT_PADDED) != 0;
    b->options = options;
    b->sshift = (options & JPEG_SCALE_HALF) ? 1 : (options & JPEG_SCALE_QUARTER) ? 2 : (options & JPEG_SCALE_EIGHTH) ? 3 : 0;
    b->gray_out = pixel_type >= EIGHT_BIT_GRAYSCALE;
    b->ptclass = (pixel_type == RGB8888) ? JD_PT_8888 : (b->gray_out ? JD_PT_GRAY : JD_PT_565);
    b->dither_bits = (pixel_type == FOUR_BIT_DITHERED) ? 4 : (pixel_type == TWO_BIT_DITHERED) ? 2 : (pixel_type == ONE_BIT_DITHERED) ? 1 : 0;
    b->resize = P.out_sizes != nullptr || P.windows != nullptr;
    b->rs_filter = filter;
    b->window = P.windows != nullptr;
    if (b->window) {
        b->wn_plans.assign(nv, JDWindowPlan{});
        b->wn_full.assign(2 * (size_t)nv, 0); b->wn_out.assign(2 * (size_t)nv, 0);
        b->wn_win.assign(P.windows, P.windows + 4 * (size_t)nv);
    }
    if (b->resize) {
        b->rs_plans.assign(nv, JDResizePlan{});
        b->rs_src_w.assign(nv, 0); b->rs_src_h.assign(nv, 0); b->rs_scratch.assign(nv, 0);
    }
    b->box = P.boxes != nullptr || P.gaps != nullptr;
    if (b->box) b->bx_plans.assign(nv, JDBoxPlan{});
    b->color = P.color != nullptr;
    if (b->color) { b->co_plans.assign(nv, JDColorPlan{}); b->co_blur.assign(nv, JDBlurPlan{}); b->co_aug.assign(nv, JDAugPlan{}); b->co_rs.assign(nv, JDResamplePlan{}); b->bl_scratch.assign(nv, 0); b->co_bgr.assign(nv, 0); }
    if (b->color && P.warp) b->co_warp.assign(nv, JDWarpPlan{});
    b->lj = (options & JPEGB200_OPT_LIBJPEG) != 0;
    if (b->lj) { b->lj_desc.assign(nv, JDLjDesc{}); b->lj_plane.assign(nv, 0); }
    b->tensor = P.spec != nullptr;
    if (b->tensor) {
        b->tn_spec = *P.spec;
        b->tn_swap.assign(nv, 0); b->tn_stage.assign(nv, 0); b->tn_plane.assign(nv, 0);
        std::vector<uint8_t> tb(3 * 256 * 4);
        b->tn_elt = jd_tensor_table(P.spec, tb.data());
        b->tn_table.assign(3 * 256, 0u);
        for (int k = 0; k < 3 * 256; k++) memcpy(&b->tn_table[k], tb.data() + (size_t)k * b->tn_elt, (size_t)b->tn_elt);
        b->tn_nc = b->ptclass == JD_PT_8888 ? 3 : 1;
        b->tn_bpp = bytes_per_pixel_class(b->ptclass);
        b->tn_planes = P.spec->layout == JPEGB200_LAYOUT_CHW ? b->tn_nc : 1;
    }
    b->infos.resize(n);
    b->parse_status.assign(nv, JPEG_SUCCESS);
    b->datas.assign(P.datas, P.datas + n);
    b->sizes.assign(P.sizes, P.sizes + n);
    b->descs.resize(nv);
    b->fdescs.resize(n);
    b->vfile.resize(nv);
    for (int f = 0, i = 0; f < n; f++) for (int k = 0; k < P.views[f]; k++) b->vfile[i++] = f;
    b->quant.assign((size_t)nv * 192, 0);   /* per view: the IDCT kernels index it by their descriptor's index */
    b->outs.assign(nv, nullptr);
    b->pitches.assign(nv, 0);
    b->comp_off.assign(n, 0);
    b->arena_off.assign(nv, 0);
    b->pplane.assign(n, 0);
}

/* input layout: one span if the files already sit back to back in host memory.  Writes contiguous_in, comp_off and
 * comp_total; 0 with a message for a batch of 3 GiB or more. */
static int layout_input(JPEGB200_BATCH *b)
{
    const int n = b->nf;
    const std::vector<const uint8_t *> &datas = b->datas;
    const std::vector<int32_t> &sizes = b->sizes;
    bool contig = true;
    for (int i = 1; i < n && contig; i++) {
        const uint8_t *prev_end = datas[i - 1] + sizes[i - 1];
        if (datas[i] < prev_end || (size_t)(datas[i] - prev_end) > 4096) contig = false;
    }
    b->contiguous_in = contig;
    size_t off = 0;
    for (int i = 0; i < n; i++) {
        if (contig) off = (size_t)(datas[i] - datas[0]);
        b->comp_off[i] = off;
        if (!contig) off += ((size_t)sizes[i] + 15) & ~(size_t)15;
    }
    b->comp_total = contig ? (size_t)(datas[n - 1] + sizes[n - 1] - datas[0]) : off;
    if (b->comp_total >= (3ull << 30)) {
        /* byte offsets into the batch buffer (and into the un-stuffed copy, which adds 32 bytes per segment) are 32-bit */
        snprintf(g_err, sizeof(g_err), "batch holds %zu compressed bytes; one job takes at most 3 GiB (JPEGB200_decodeBatch splits larger batches)", b->comp_total);
        return 0;
    }
    return 1;
}

/* header parse (of the thumbnail with JPEG_EXIF_THUMBNAIL), progressive mode and the per-file refusals.  Writes infos[f],
 * and P.fscans / P.ftabs for a file decoded from all its scans. */
static FileAdmit admit_file(JPEGB200_BATCH *b, CreatePlan &P, int f)
{
    FileAdmit a;
    JDInfo &inf = b->infos[f];
    const uint8_t *data = P.datas[f];
    const int size = P.sizes[f], options = b->options;
    int ok = jd_parse_header_opt(data, size, 0, &inf, options);
    int st = ok ? JPEG_SUCCESS : inf.error;
    if (ok && (options & JPEG_EXIF_THUMBNAIL)) {
        if (inf.thumb_data == 0 || inf.thumb_w == 0) { ok = 0; st = JPEG_INVALID_PARAMETER; }
        else { ok = jd_parse_header_opt(data, size, inf.thumb_data, &inf, options); if (!ok) st = inf.error; }
    }
    if (ok && inf.mode == 0xC2 && (options & JPEGB200_OPT_PROGRESSIVE)) {
        a.nsc = jd_prog_parse(data, size, (options & JPEG_EXIF_THUMBNAIL) ? inf.thumb_data : 0, &inf, P.fscans.data(),
                              P.ftabs.data(), &a.ntb);
        if (a.nsc <= 0) { ok = 0; st = -a.nsc; } else a.full = true;
    } else if (ok && inf.mode == 0xC2) {
        /* progressive: like the reference, only the DC coefficients of the first scan are decoded and a 1/8-size image
         * is produced (jpeg.inl:4964-4966, JPEGDecodeMCU_P :1819-1884).  That needs a first scan that is the interleaved
         * DC scan of every component (Ss = Se = 0, Ah = 0) -- what every common encoder writes -- and 1/8 scale. */
        a.prog = true;
        if (b->sshift != 3 || inf.p.ncomp_in_scan != inf.ncomp || inf.p.scan_start != 0 || inf.p.scan_end != 0 || (inf.approx >> 4) != 0 ||
            (inf.approx & 15) > 13) { ok = 0; st = JPEG_UNSUPPORTED_FEATURE; }
    } else if (ok && inf.mode != 0xC0) { ok = 0; st = JPEG_UNSUPPORTED_FEATURE; }
    if (ok && !a.full && !inf.tables_ok) { ok = 0; st = JPEG_DECODE_ERROR; }  /* jpeg.inl:2166 */
    if (ok && inf.ncomp == 1 && b->pixel_type == RGB8888 && !b->lj) { ok = 0; st = JPEG_INVALID_PARAMETER; }
    if (ok && b->lj && b->pixel_type == EIGHT_BIT_GRAYSCALE && !jd_lj_is_ycc(&inf)) { ok = 0; st = JPEG_UNSUPPORTED_FEATURE; }
    if (ok && (uint64_t)size >= (512ull << 20)) { ok = 0; st = JPEG_UNSUPPORTED_FEATURE; }   /* image-relative record indices are 32-bit */
    a.ok = ok; a.status = st;
    return a;
}

/* the transform of each of the file's views v0 .. v0 + nvf - 1.  Writes exif_tag, orient and P.ks. */
static void resolve_orients(JPEGB200_BATCH *b, CreatePlan &P, int f, int v0, int nvf)
{
    const JDInfo &inf = b->infos[f];
    for (int i = v0; i < v0 + nvf; i++) {
        b->exif_tag[i] = inf.orientation;
        if (P.orients) {
            /* 0: the file's tag (none or out of range: identity); 1-8: that transform; anything else is refused by jd_views_plan */
            const int k = P.orients[i] == 0 ? ((inf.orientation >= 1 && inf.orientation <= 8) ? inf.orientation : 1) : P.orients[i];
            if (k <= 8) b->orient[i] = (uint8_t)k;
            P.ks[i] = (uint8_t)k;
        }
    }
}

/* the walk of a file after some of its views were refused late (box, colour operations): without a rectangle every view
 * walks the whole file, with rectangles the deepest valid view sets it */
static uint32_t kept_walk(const JPEGB200_BATCH *b, const CreatePlan &P, int v0, int nvf, uint32_t walk)
{
    uint32_t kept = 0;
    for (int i = v0; i < v0 + nvf; i++) {
        const uint32_t w = b->roi ? (uint32_t)b->plans[i].nseg_walk : walk;
        if (P.vok[i] && w > kept) kept = w;
    }
    return kept;
}

/* The views' own arguments (no such transform, a rectangle outside the output, a resize target outside 1..65535) and how
 * deep the file is walked: down to the deepest last MCU row among its valid views.  Writes plans, P.srects and P.vok;
 * returns the restart intervals to walk, 0 when no view is valid. */
/* With windows, before the views are planned: each view's full S (what the call without windows resizes), its window plan,
 * and the rectangle it decodes: its support, inside the caller's rectangle (boxed views keep the whole S).  A view whose
 * own arguments are refused keeps them, so that jd_views_plan refuses it; a refused window clears wn_ok. */
static void plan_windows(JPEGB200_BATCH *b, CreatePlan &P, int f, int v0, int nvf, std::vector<int32_t> &wn_ok)
{
    const JDInfo &inf = b->infos[f];
    for (int i = v0; i < v0 + nvf; i++) {
        int32_t *r = &P.wn_rois[4 * (size_t)i];
        const int32_t *cr = P.caller_rois ? P.caller_rois + 4 * (size_t)i : nullptr;
        const int s = P.draft ? jd_draft_shift(P.draft[i]) : b->sshift;
        const int k = P.orients ? P.ks[i] : 1;
        int W = (inf.width + (1 << (s < 0 ? 0 : s)) - 1) >> (s < 0 ? 0 : s), H = (inf.height + (1 << (s < 0 ? 0 : s)) - 1) >> (s < 0 ? 0 : s);
        if (k >= 5 && k <= 8) std::swap(W, H);
        if (cr) { r[0] = cr[0]; r[1] = cr[1]; r[2] = cr[2]; r[3] = cr[3]; }
        else { r[0] = 0; r[1] = 0; r[2] = W; r[3] = H; }
        const bool ok = s >= 0 && k >= 1 && k <= 8 && r[0] >= 0 && r[1] >= 0 && r[2] >= 1 && r[3] >= 1 &&
                        (int64_t)r[0] + r[2] <= W && (int64_t)r[1] + r[3] <= H;
        const int32_t sw = ok ? r[2] : 1, sh = ok ? r[3] : 1;
        b->wn_full[2 * (size_t)i] = sw; b->wn_full[2 * (size_t)i + 1] = sh;
        if (P.wn_sizes.size()) { P.wn_sizes[2 * (size_t)i] = sw; P.wn_sizes[2 * (size_t)i + 1] = sh; }
        wn_ok[i - v0] = 1;
        b->wn_out[2 * (size_t)i] = P.out_sizes[2 * (size_t)i]; b->wn_out[2 * (size_t)i + 1] = P.out_sizes[2 * (size_t)i + 1];
        if (b->box || !ok) continue;   /* a box reads all of S; a refused view is refused by jd_views_plan */
        const int32_t *os = &P.out_sizes[2 * (size_t)i];
        if (os[0] < 1 || os[1] < 1 || os[0] > 65535 || os[1] > 65535) continue;
        JDWindowPlan &wp = b->wn_plans[i];
        if (!jd_window_plan(sw, sh, os[0], os[1], b->rs_filter, P.windows + 4 * (size_t)i, bytes_per_pixel_class(b->ptclass), &wp)) {
            wn_ok[i - v0] = 0;
            continue;
        }
        r[0] += wp.sx; r[1] += wp.sy; r[2] = wp.sw; r[3] = wp.sh;
    }
}

static uint32_t plan_views(JPEGB200_BATCH *b, CreatePlan &P, int f, int v0, int nvf)
{
    const JDInfo &inf = b->infos[f];
    uint32_t walk = 0;
    std::vector<int32_t> wn_ok;
    if (b->window) { wn_ok.assign((size_t)nvf, 1); plan_windows(b, P, f, v0, nvf, wn_ok); }
    if (!P.draft) {
        walk = (uint32_t)jd_views_plan(inf.width, inf.height, inf.subsample, inf.restart_interval, b->sshift, nvf,
                                       P.rois ? P.rois + 4 * (size_t)v0 : nullptr, P.orients ? &P.ks[v0] : nullptr,
                                       P.out_sizes ? P.out_sizes + 2 * (size_t)v0 : nullptr, &b->plans[v0], &P.srects[4 * (size_t)v0],
                                       &P.vok[v0]);
    } else {
        /* each view at its own scale (a libjpeg batch walks at full scale: b->sshift is 0); an unknown denominator
         * invalidates that view alone */
        for (int i = v0; i < v0 + nvf; i++) {
            const int sh = jd_draft_shift(P.draft[i]);
            const uint32_t w = (uint32_t)jd_views_plan(inf.width, inf.height, inf.subsample, inf.restart_interval, sh < 0 ? 0 : sh, 1,
                                                       P.rois ? P.rois + 4 * (size_t)i : nullptr, P.orients ? &P.ks[i] : nullptr,
                                                       P.out_sizes ? P.out_sizes + 2 * (size_t)i : nullptr, &b->plans[i],
                                                       &P.srects[4 * (size_t)i], &P.vok[i]);
            if (sh < 0) { P.vok[i] = 0; continue; }
            b->lj_desc[i].shift = (uint32_t)sh;
            if (w > walk) walk = w;
        }
    }
    if (walk != 0 && b->window) {
        bool dropped = false;
        for (int i = v0; i < v0 + nvf; i++) if (P.vok[i] && !wn_ok[i - v0]) { P.vok[i] = 0; dropped = true; }
        if (dropped) walk = kept_walk(b, P, v0, nvf, walk);
    }
    if (walk != 0 && b->lj && b->roi) {
        /* what libjpeg's fancy upsampling reads around each rectangle */
        walk = 0;
        for (int i = v0; i < v0 + nvf; i++) {
            if (!P.vok[i]) continue;
            const int32_t *sr = &P.srects[4 * (size_t)i];
            const int32_t r[4] = {sr[0], sr[1], P.orients ? sr[2] : P.rois[4 * (size_t)i + 2], P.orients ? sr[3] : P.rois[4 * (size_t)i + 3]};
            jd_lj_plan_extend_s(inf.width, inf.height, inf.subsample, inf.restart_interval, (int)b->lj_desc[i].shift, r, &b->plans[i]);
            if ((uint32_t)b->plans[i].nseg_walk > walk) walk = (uint32_t)b->plans[i].nseg_walk;
        }
    }
    if (walk != 0 && b->box) {
        /* each valid view's box and gap on S, its output before the resize; a refused view leaves the walk to the others */
        bool dropped = false;
        for (int i = v0; i < v0 + nvf; i++) {
            if (!P.vok[i]) continue;
            const int s = b->lj ? (int)b->lj_desc[i].shift : b->sshift;
            const int sw = b->roi ? b->plans[i].out_w : (inf.width + (1 << s) - 1) >> s;
            const int sh = b->roi ? b->plans[i].out_h : (inf.height + (1 << s) - 1) >> s;
            const double whole[4] = {0.0, 0.0, (double)sw, (double)sh};
            if (!jd_box_plan(sw, sh, P.out_sizes[2 * (size_t)i], P.out_sizes[2 * (size_t)i + 1], b->rs_filter,
                             P.boxes ? P.boxes + 4 * (size_t)i : whole, P.gaps ? P.gaps[i] : 0.0, bytes_per_pixel_class(b->ptclass),
                             &b->bx_plans[i]) ||
                (b->window && !jd_window_box(&b->bx_plans[i], P.out_sizes[2 * (size_t)i], P.out_sizes[2 * (size_t)i + 1],
                                             P.windows + 4 * (size_t)i, bytes_per_pixel_class(b->ptclass), &b->wn_plans[i]))) {
                P.vok[i] = 0;
                dropped = true;
            }
        }
        if (dropped) walk = kept_walk(b, P, v0, nvf, walk);
    }
    if (walk != 0 && b->color) {
        /* each valid view's operations; one Pillow or torchvision refuses leaves the walk to the others */
        bool dropped = false;
        for (int i = v0; i < v0 + nvf; i++) {
            if (!P.vok[i]) continue;
            /* the view's final size, which the geometric ops' mappings depend on (padded output takes no operations) */
            const int s = b->lj ? (int)b->lj_desc[i].shift : b->sshift;
            uint32_t w = b->resize ? (uint32_t)P.out_sizes[2 * (size_t)i] : b->roi ? (uint32_t)b->plans[i].out_w : (uint32_t)((inf.width + (1 << s) - 1) >> s);
            uint32_t h = b->resize ? (uint32_t)P.out_sizes[2 * (size_t)i + 1] : b->roi ? (uint32_t)b->plans[i].out_h : (uint32_t)((inf.height + (1 << s) - 1) >> s);
            if (b->window) { w = (uint32_t)P.windows[4 * (size_t)i + 2]; h = (uint32_t)P.windows[4 * (size_t)i + 3]; }
            if (!jd_color_plan_warp(P.color + JPEGB200_COLOR_MAX_OPS * (size_t)i, P.warp ? P.warp + JPEGB200_COLOR_MAX_OPS * (size_t)i : nullptr,
                                    b->ptclass == JD_PT_GRAY, w, h, &b->co_plans[i], &b->co_blur[i], &b->co_aug[i], &b->co_rs[i],
                                    P.warp ? &b->co_warp[i] : nullptr)) {
                P.vok[i] = 0;
                dropped = true;
            }
        }
        if (dropped) walk = kept_walk(b, P, v0, nvf, walk);
    }
    return walk;
}

/* restart segments and chunks of the file (none when it is not walked), and the refusal of a file whose records would not
 * fit 32-bit image-relative indices */
static void size_file_walk(const JPEGB200_BATCH *b, int f, FileAdmit &a)
{
    const JDInfo &inf = b->infos[f];
    const int size = b->sizes[f];
    a.total_mcus = a.ok ? (uint32_t)inf.mcus_x * inf.mcus_y : 0u;
    a.mps = inf.restart_interval ? (uint32_t)inf.restart_interval : a.total_mcus;
    a.nseg = (a.ok && !a.full) ? (a.total_mcus + a.mps - 1) / a.mps : 0u;   /* a full progressive file has walkers instead */
    /* no restart markers: one long dependent stream -> chunk-parallel decode */
    a.nch = (a.ok && !a.prog && inf.restart_interval == 0 && a.nseg == 1 && size - inf.scan_offset >= 4096)
                ? ((uint32_t)(size - inf.scan_offset) + JD_CHUNK_BYTES - 1) / JD_CHUNK_BYTES + 1 : 0u;
    if (a.ok && jd_rec_extent((uint64_t)size, (uint32_t)inf.scan_offset, a.nseg, a.nch) > (1ull << 32)) {
        a.ok = 0; a.status = JPEG_UNSUPPORTED_FEATURE;   /* its record indices would wrap onto its own first records */
    }
}

/* a file that is not walked: harmless empty descriptors for it and its views */
static void fill_refused_descs(JPEGB200_BATCH *b, const CreatePlan &P, int f, int v0, int nvf, int status)
{
    JDImageDesc &d = b->fdescs[f];
    d.nseg = 0; d.seg_base = P.seg; d.blk_base = (uint32_t)P.blk; d.status = (uint32_t)status;
    for (int i = v0; i < v0 + nvf; i++) {
        b->descs[i] = d;
        b->descs[i].status = (uint32_t)b->parse_status[i];
    }
}

/* kernels read quant column-major ([c * 8 + r]) so a lane's column is one 16-byte load; one copy per view */
static void fill_quant(JPEGB200_BATCH *b, int f, int v0, int nvf)
{
    const JDInfo &inf = b->infos[f];
    int16_t qn[192];
    jd_build_quant(&inf, qn);
    for (int i = v0; i < v0 + nvf; i++) {
        int32_t *qt = &b->quant[(size_t)i * 192];
        if (b->lj) { jd_lj_quant(&inf, qt); continue; }   /* islow dequantizes with the raw DQT values */
        for (int cc = 0; cc < 3; cc++)
            for (int nn = 0; nn < 64; nn++) qt[cc * 64 + (nn & 7) * 8 + (nn >> 3)] = qn[cc * 64 + nn];
    }
}

/* Huffman LUT set of the file: dedupe on the raw DHT content.  Appends to luts; counts a hit of the context's shared table. */
static uint32_t lut_set_for(JPEGB200_BATCH *b, CreatePlan &P, int f)
{
    JPEGB200_CTX *ctx = b->ctx;
    const JDInfo &inf = b->infos[f];
    uint32_t li = 0;
    const uint64_t h = jd_tables_hash(&inf);
    for (; li < P.lut_hash.size(); li++) if (P.lut_hash[li] == h && jd_tables_equal(&inf, &b->infos[P.lut_owner[li]])) break;
    const bool shared = ctx->has_shared && ctx->shared_hash == h && ctx->shared_hash2 == jd_tables_hash2(&inf);
    if (li == P.lut_hash.size()) {
        P.lut_hash.push_back(h); P.lut_owner.push_back(f);
        b->luts.resize((size_t)(li + 1) * JD_LUT_ENTRIES);
        if (shared) memcpy(&b->luts[(size_t)li * JD_LUT_ENTRIES], ctx->shared_lut, JD_LUT_ENTRIES * 2);
        else jd_build_lut(&inf, &b->luts[(size_t)li * JD_LUT_ENTRIES]);
    }
    if (shared) ctx->shared_hits++;
    return li;
}

/* the entropy-facing descriptor of an admitted file; a restart-free file joins the chunk list (nchunks, max_nch, cimg_list) */
static void fill_file_desc(JPEGB200_BATCH *b, const CreatePlan &P, int f, const FileAdmit &a, uint32_t walk, uint32_t lutset)
{
    const JDInfo &inf = b->infos[f];
    JDImageDesc &d = b->fdescs[f];
    d.scan_off = (uint32_t)(b->comp_off[f] + inf.scan_offset);
    d.scan_end = (uint32_t)(b->comp_off[f] + b->sizes[f]);
    d.width = (uint16_t)inf.width; d.height = (uint16_t)inf.height;
    d.mcus_x = (uint16_t)inf.mcus_x; d.mcus_y = (uint16_t)inf.mcus_y;
    d.subsample = (uint8_t)inf.subsample; d.ncomp = (uint8_t)inf.ncomp; d.bpm = (uint8_t)inf.bpm; d.tsel = (uint8_t)inf.tsel;
    d.mcus_per_seg = a.mps;
    d.nseg = a.nseg;
    d.nseg_walk = a.full ? 0u : b->roi ? walk : d.nseg;   /* a full progressive file has no restart segments to walk */
    d.chunk_base = 0; d.nch = 0;
    d.prog = a.prog ? (1u | ((uint32_t)(inf.approx & 15) << 8)) : 0u;
    if (a.nch) {
        d.chunk_base = b->nchunks;
        d.nch = a.nch;
        b->nchunks += d.nch;
        if (d.nch > b->max_nch) b->max_nch = d.nch;
        b->cimg_list.push_back((uint32_t)f);
    }
    d.seg_base = P.seg;
    d.blk_base = (uint32_t)P.blk;
    d.lutset = lutset;
    /* coefficient records: image-relative indices (jd_core.h JD_REC_INDEX), one slot per restart segment and per chunk */
    d.comp_off = (uint32_t)b->comp_off[f];
    d.rec_base = P.rec_total;
}

/* a file decoded from all its scans: its walkers (pscans) down to the deepest MCU row a valid view needs, its record cap
 * (pfiles, P.rec_total), its coefficient plane (pplane) and its tables, de-duplicated on content (ptabs) */
static void add_prog_file(JPEGB200_BATCH *b, CreatePlan &P, int f, int v0, int nvf, const FileAdmit &a)
{
    const JDInfo &inf = b->infos[f];
    uint32_t rows = (uint32_t)inf.mcus_y;
    if (b->roi) {
        rows = 0;
        for (int i = v0; i < v0 + nvf; i++) if (P.vok[i] && (uint32_t)b->plans[i].mcu_y1 + 1u > rows) rows = (uint32_t)b->plans[i].mcu_y1 + 1u;
    }
    const uint64_t cap = jd_prog_rec_cap((uint64_t)b->sizes[f], (uint32_t)a.nsc);   /* records sized by jd_prog_rec_cap */
    /* whole 16-byte chunks: the entropy walk of the next image stores its records as aligned 16-byte chunks */
    P.rec_total += (cap + 15u) & ~(uint64_t)7;
    b->pfiles.push_back(JDProgFile{cap, (uint32_t)f, rows});
    b->pplane[f] = (int64_t)a.total_mcus * inf.bpm * 128;
    b->pplane_total += b->pplane[f];
    for (int k = 0; k < a.nsc; k++) {
        JDProgScan s = P.fscans[k];
        s.start += (uint32_t)b->comp_off[f]; s.end += (uint32_t)b->comp_off[f];
        s.img = (uint32_t)f;
        s.row_limit = rows;
        const int ntab = (s.ss == 0 && s.ah != 0) ? 0 : s.ncs;   /* DC refinements read raw bits */
        for (int i = 0; i < ntab; i++) {
            const JDProgHuff &t = P.ftabs[s.tab[i]];
            uint64_t th = 1469598103934665603ull;
            for (size_t q = 0; q < sizeof(t); q++) th = (th ^ ((const uint8_t *)&t)[q]) * 1099511628211ull;
            std::vector<uint32_t> &same = P.ptab_index[th];
            size_t q = 0;
            while (q < same.size() && memcmp(&b->ptabs[same[q]], &t, sizeof(t)) != 0) q++;
            if (q == same.size()) { same.push_back((uint32_t)b->ptabs.size()); b->ptabs.push_back(t); }
            s.tab[i] = same[q];
        }
        b->pscans.push_back(s);
    }
}

/* View i of admitted file f: the file's descriptor (its walk, blocks and records) with the view's rectangle, orientation and
 * output.  Writes descs[i], pitches[i], arena_off[i] and the view's libjpeg box, resize plan + scratch and tensor staging;
 * advances P.out_total / P.gray_total.  roi_mcu_end goes into the view's descriptor only: jdk_stitch reports the file's
 * first error, jd_view_err_mcu (JPEGB200_batchErrMcu) judges it per view.  0 with a message when the resize cannot be
 * planned. */
static int plan_view_output(JPEGB200_BATCH *b, CreatePlan &P, int f, int i)
{
    const JDInfo &inf = b->infos[f];
    const int s = b->lj ? (int)b->lj_desc[i].shift : b->sshift;   /* a libjpeg batch scales per view (draft) */
    JDImageDesc &vd = b->descs[i];
    if (b->parse_status[i] != JPEG_SUCCESS) {   /* an invalid view of a walked file: empty, like a refused image */
        memset(&vd, 0, sizeof(vd));
        vd.seg_base = P.seg; vd.blk_base = (uint32_t)P.blk; vd.status = (uint32_t)b->parse_status[i];
        return 1;
    }
    vd = b->fdescs[f];
    vd.out_w = (uint32_t)((inf.width + (1 << s) - 1) >> s);
    vd.out_h = (uint32_t)((inf.height + (1 << s) - 1) >> s);
    if (b->padded) {
        vd.out_w = (uint32_t)inf.mcus_x * (uint32_t)(inf.mcu_w >> s);
        vd.out_h = (uint32_t)inf.mcus_y * (uint32_t)(inf.mcu_h >> s);
    }
    if (b->roi) {
        const JDRoiPlan &pl = b->plans[i];
        vd.out_w = (uint32_t)pl.out_w; vd.out_h = (uint32_t)pl.out_h;
        vd.roi_x = (uint16_t)P.srects[4 * (size_t)i]; vd.roi_y = (uint16_t)P.srects[4 * (size_t)i + 1];
        vd.mcu_x0 = (uint16_t)pl.mcu_x0; vd.mcu_y0 = (uint16_t)pl.mcu_y0;
        vd.roi_mcu_end = (uint32_t)pl.mcu_end;
        vd.orient = P.orients ? b->orient[i] : 0u;
    }
    if (b->lj) {
        /* the MCU box whose planes jdk_lj_idct writes: the rectangle's, extended by jd_lj_plan_extend */
        JDLjDesc &L = b->lj_desc[i];
        L.mx0 = b->roi ? (uint32_t)b->plans[i].mcu_x0 : 0u; L.my0 = b->roi ? (uint32_t)b->plans[i].mcu_y0 : 0u;
        L.nmx = b->roi ? (uint32_t)(b->plans[i].mcu_x1 - b->plans[i].mcu_x0 + 1) : (uint32_t)inf.mcus_x;
        L.nmy = b->roi ? (uint32_t)(b->plans[i].mcu_y1 - b->plans[i].mcu_y0 + 1) : (uint32_t)inf.mcus_y;
        L.ycc = (uint32_t)jd_lj_is_ycc(&inf);
        const uint64_t blocks = (uint64_t)L.nmx * L.nmy * (uint64_t)inf.bpm;
        const uint64_t px = (uint64_t)vd.out_w * vd.out_h;
        if (L.shift == 0) {
            b->lj_plane[i] = (int64_t)align256(blocks * 64u);
            if (blocks > b->lj_max_blocks) b->lj_max_blocks = (uint32_t)blocks;
            if (px > b->lj_max_pixels) b->lj_max_pixels = (uint32_t)px;
        } else {
            /* size_c x size_c samples per block of each component (jd_ljpeg.h) */
            const uint32_t hs = (inf.subsample >> 4) ? (uint32_t)(inf.subsample >> 4) : 1u, vs = (inf.subsample & 15) ? (uint32_t)(inf.subsample & 15) : 1u;
            const uint64_t ys = 8u >> L.shift, cs = jd_lj_csize(L.shift, hs, vs);
            const uint64_t per_mcu = hs * vs * ys * ys + (uint64_t)(inf.ncomp - 1) * cs * cs;
            b->lj_plane[i] = (int64_t)align256((uint64_t)L.nmx * L.nmy * per_mcu);
            if (blocks > b->lj_s_blocks[L.shift]) b->lj_s_blocks[L.shift] = (uint32_t)blocks;
            if (px > b->lj_s_pixels[L.shift]) b->lj_s_pixels[L.shift] = (uint32_t)px;
        }
        b->lj_plane_total += b->lj_plane[i];
    }
    if (b->resize) {
        /* S = what the same call without out_sizes stores; the descriptor carries the resized size from here on */
        const int bp = bytes_per_pixel_class(b->ptclass);
        JDResizePlan &rp = b->rs_plans[i];
        int32_t rw = P.out_sizes[2 * (size_t)i], rh = P.out_sizes[2 * (size_t)i + 1];
        if (b->window) {   /* planned by plan_windows (or with the box by plan_views); S is the support */
            rp = b->wn_plans[i].rp;
            rw = P.windows[4 * (size_t)i + 2]; rh = P.windows[4 * (size_t)i + 3];
        } else if (b->box) rp = b->bx_plans[i].rp;   /* planned with the box by plan_views */
        else if (!jd_resize_plan((int)vd.out_w, (int)vd.out_h, rw, rh, b->rs_filter, bp, &rp)) {
            snprintf(g_err, sizeof(g_err), "resize plan failed for image %d", i);
            return 0;
        }
        b->rs_src_w[i] = vd.out_w; b->rs_src_h[i] = vd.out_h;
        b->rs_scratch[i] = (int64_t)align256((size_t)vd.out_w * vd.out_h * bp) + (int64_t)align256((size_t)rp.mid_bytes);
        if (b->box && (b->bx_plans[i].fx > 1 || b->bx_plans[i].fy > 1))   /* the reduced image */
            b->rs_scratch[i] += (int64_t)align256((size_t)b->bx_plans[i].rw * b->bx_plans[i].rh * bp);
        b->rs_scratch_total += b->rs_scratch[i];
        vd.out_w = (uint32_t)rw; vd.out_h = (uint32_t)rh;
    }
    if (b->tensor) {
        /* U = what the same call without spec stores (out_w x out_h); staged, then converted */
        b->tn_stage[i] = (int64_t)align256((size_t)vd.out_w * vd.out_h * b->tn_bpp);
        b->tn_stage_total += b->tn_stage[i];
        /* a libjpeg decode stores R, G, B for every file */
        const bool bgr = !b->lj && jd_rgb8888_is_bgr(b->ctx->arith, b->sshift, inf.ncomp, inf.subsample) != 0;
        b->tn_swap[i] = (uint8_t)(b->tn_nc == 3 && bgr != (b->tn_spec.bgr != 0));
    }
    if (b->color) {   /* the colour operations read true R, G, B: a libjpeg decode stores R, G, B for every file */
        b->co_bgr[i] = (uint8_t)(b->ptclass == JD_PT_8888 && !b->lj && jd_rgb8888_is_bgr(b->ctx->arith, b->sshift, inf.ncomp, inf.subsample));
        const JDColorPlan &cp = b->co_plans[i];
        bool own = false;
        int64_t nlut = 0;
        uint64_t jq = 0;   /* a JPEG op on an RGB view: its decoded planes (a gray view's blocks are written back in place) */
        for (uint32_t k = 0; k < cp.nops; k++) {
            if (JD_CO_JQ(cp.op[k])) {
                uint32_t hs, vs;
                jd_jq_factors(cp.op[k], &hs, &vs);
                if (b->ptclass != JD_PT_GRAY) jq = std::max(jq, jd_jq_scratch(jd_jq_geo(vd.out_w, vd.out_h, hs, vs)));
            } else own = own || JD_CO_OWN_KERNEL(cp.op[k]);
            nlut += JD_CO_LUT(cp.op[k]) ? 1 : 0;
        }
        if (own) b->bl_scratch[i] = (int64_t)align256((size_t)vd.out_w * vd.out_h * bytes_per_pixel_class(b->ptclass));
        if ((int64_t)align256((size_t)jq) > b->bl_scratch[i]) b->bl_scratch[i] = (int64_t)align256((size_t)jq);
        b->bl_scratch[i] += nlut * JD_AU_HIST * (int64_t)sizeof(unsigned long long);
        b->bl_scratch_total += b->bl_scratch[i];
    }
    size_t pitch;
    if (b->tensor) pitch = (size_t)vd.out_w * (b->tn_spec.layout == JPEGB200_LAYOUT_HWC ? b->tn_nc : 1) * b->tn_elt;
    else if (b->dither_bits) {
        const uint32_t pw = (uint32_t)inf.mcus_x * (uint32_t)(inf.mcu_w >> s);
        pitch = ((size_t)pw * b->dither_bits + 7) / 8;
        P.gray_total += align256((size_t)pw * (size_t)inf.mcus_y * (size_t)(inf.mcu_h >> s));
    } else pitch = (size_t)vd.out_w * bytes_per_pixel_class(b->ptclass);
    vd.out_pitch = (uint32_t)pitch;
    b->pitches[i] = (int64_t)pitch;
    b->arena_off[i] = P.out_total;
    P.out_total += align256(pitch * vd.out_h * (b->tensor ? (size_t)b->tn_planes : 1u));
    return 1;
}

/* one launch per wave of scan walkers; inside a wave the longest scans start first.  Sorts pscans, writes pwave_off. */
static void sort_prog_waves(JPEGB200_BATCH *b)
{
    if (b->pscans.empty()) return;
    std::stable_sort(b->pscans.begin(), b->pscans.end(), [](const JDProgScan &x, const JDProgScan &y) {
        return x.wave != y.wave ? x.wave < y.wave : (x.end - x.start) > (y.end - y.start);
    });
    for (size_t k = 0; k < b->pscans.size(); k++)
        while (b->pwave_off.size() <= b->pscans[k].wave) b->pwave_off.push_back((uint32_t)k);
    b->pwave_off.push_back((uint32_t)b->pscans.size());
}

/* Work list (work, cta_lut, seg_img): CTAs of 128 segments sharing one LUT set.  With a region of interest the restart
 * intervals that start below its last MCU row are left out, but every interval above it stays in: the reference's
 * bit-window phase is carried from one interval to the next (SURVEY.md fact 4, A.2), so the pixels inside the rectangle
 * depend on the walk of every interval before them.  One entry per file: its views share the walk. */
static void build_work_list(JPEGB200_BATCH *b)
{
    b->seg_img.resize(b->nseg ? b->nseg : 1);
    const std::vector<JDImageDesc> &fd = b->fdescs;
    for (uint32_t li = 0; li < (b->nlut ? b->nlut : 1); li++) {
        for (int i = 0; i < b->nf; i++) {
            const JDImageDesc &d = fd[i];
            if (d.nseg == 0 || d.lutset != li) continue;   /* nseg = 0: a file that is not walked */
            for (uint32_t s2 = 0; s2 < d.nseg; s2++) {
                b->seg_img[d.seg_base + s2] = (uint32_t)i;
                if (d.nch == 0 && s2 < d.nseg_walk) b->work.push_back(d.seg_base + s2);
            }
        }
        while (b->work.size() % JD_ENTROPY_THREADS) b->work.push_back(JD_NONE);
        while (b->cta_lut.size() < b->work.size() / JD_ENTROPY_THREADS) b->cta_lut.push_back(li);
    }
}

/* every file in turn: admission, its views' plans, its descriptor and tables, its views' outputs.  0 with a message when
 * the batch as a whole is refused. */
static int plan_files(JPEGB200_BATCH *b, CreatePlan &P)
{
    for (int f = 0, v0 = 0; f < b->nf; v0 += P.views[f], f++) {
        const int nvf = P.views[f];   /* the file's views (images) are v0 .. v0 + nvf - 1 */
        const JDInfo &inf = b->infos[f];
        memset(&b->fdescs[f], 0, sizeof(JDImageDesc));
        FileAdmit a = admit_file(b, P, f);
        const int file_ok = a.ok;
        resolve_orients(b, P, f, v0, nvf);
        uint32_t walk = 0;
        if (a.ok) {
            walk = plan_views(b, P, f, v0, nvf);
            if (walk == 0) a.ok = 0;   /* no valid view: the file is not walked */
        }
        size_file_walk(b, f, a);
        /* a failed parse first, then the view's own arguments, then the record extent */
        for (int i = v0; i < v0 + nvf; i++) b->parse_status[i] = (file_ok && !P.vok[i]) ? JPEG_INVALID_PARAMETER : a.status;
        if (!a.ok) { fill_refused_descs(b, P, f, v0, nvf, a.status); continue; }
        fill_quant(b, f, v0, nvf);
        const uint32_t lutset = a.full ? 0u : lut_set_for(b, P, f);   /* a full progressive file uses its scans' own tables */
        fill_file_desc(b, P, f, a, walk, lutset);
        if (a.full) add_prog_file(b, P, f, v0, nvf, a);
        else P.rec_total += (uint64_t)JD_REC_PER_BYTE * (uint64_t)(((size_t)b->sizes[f] + 15) & ~(size_t)15) + (uint64_t)JD_REC_SLOT_SLACK * (a.nseg + a.nch + 1u);
        for (int i = v0; i < v0 + nvf; i++) if (!plan_view_output(b, P, f, i)) return 0;
        P.seg += a.nseg;
        b->nseg_walk += b->fdescs[f].nseg_walk;
        P.blk += (uint64_t)a.total_mcus * inf.bpm;
        if (P.blk >= (1ull << 32)) { snprintf(g_err, sizeof(g_err), "batch too large (block count)"); return 0; }
    }
    b->nseg = P.seg; b->nblk = P.blk; b->nlut = (uint32_t)P.lut_hash.size();
    b->rec_total = P.rec_total;
    b->out_total = P.out_total; b->gray_total = P.gray_total;
    if ((uint64_t)b->comp_total + 32ull * P.seg + 4096ull >= (1ull << 32)) {
        snprintf(g_err, sizeof(g_err), "batch too large (%zu compressed bytes in %u restart segments)", b->comp_total, P.seg);
        return 0;
    }
    return 1;
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateViews(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                                     const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                                     const uint8_t *orients, const int32_t *out_sizes, int filter,
                                                     const JPEGB200_TensorSpec *spec)
{
    return JPEGB200_batchCreateDraft(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, nullptr);
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateDraft(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                                     const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                                     const uint8_t *orients, const int32_t *out_sizes, int filter,
                                                     const JPEGB200_TensorSpec *spec, const uint8_t *draft)
{
    return JPEGB200_batchCreateBox(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, draft,
                                   nullptr, nullptr);
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateBox(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                                   const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                                   const uint8_t *orients, const int32_t *out_sizes, int filter,
                                                   const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                                   const double *reducing_gaps)
{
    return JPEGB200_batchCreateColor(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, draft,
                                     boxes, reducing_gaps, nullptr);
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateColor(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                                     const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                                     const uint8_t *orients, const int32_t *out_sizes, int filter,
                                                     const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                                     const double *reducing_gaps, const JPEGB200_ColorOp *color_ops)
{
    return JPEGB200_batchCreateWarp(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, draft,
                                    boxes, reducing_gaps, color_ops, nullptr);
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateWarp(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                                    const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                                    const uint8_t *orients, const int32_t *out_sizes, int filter,
                                                    const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                                    const double *reducing_gaps, const JPEGB200_ColorOp *color_ops,
                                                    const JPEGB200_WarpArgs *warp_args)
{
    return JPEGB200_batchCreateWindow(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, draft,
                                      boxes, reducing_gaps, color_ops, warp_args, nullptr);
}

extern "C" JPEGB200_BATCH *JPEGB200_batchCreateWindow(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                                      const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                                      const uint8_t *orients, const int32_t *out_sizes, int filter,
                                                      const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                                      const double *reducing_gaps, const JPEGB200_ColorOp *color_ops,
                                                      const JPEGB200_WarpArgs *warp_args, const int32_t *windows)
{
    if (!ctx) { snprintf(g_err, sizeof(g_err), "invalid parameter"); return nullptr; }
    int64_t nv = 0;   /* images of the batch: views */
    /* a window resizes (to S's own size without out_sizes): the resize's refusals (RGB565, dithered, padded) apply, named
     * for the windows */
    const int rs_filter = out_sizes ? filter : JPEGB200_RESIZE_BILINEAR;
    if (windows) {
        const int pt = jd_fold_luma_only(pixel_type, options);
        const char *why = (pt == RGB565_LITTLE_ENDIAN || pt == RGB565_BIG_ENDIAN) ? "RGB565 pixel types"
                          : (pt >= FOUR_BIT_DITHERED && pt <= ONE_BIT_DITHERED) ? "dithered pixel types"
                          : (options & JPEGB200_OPT_PADDED) ? "padded output" : nullptr;
        if (why) { snprintf(g_err, sizeof(g_err), "windows are not supported with %s", why); return nullptr; }
    }
    if (!jd_check_batch_features(pixel_type, options, n, views, rois != nullptr, orients != nullptr,
                                 out_sizes != nullptr || windows != nullptr, rs_filter, spec, &nv, g_err, (int)sizeof(g_err)) ||
        !jd_check_draft(options, draft, g_err, (int)sizeof(g_err)) || !jd_check_box(out_sizes, boxes, reducing_gaps, g_err, (int)sizeof(g_err)) ||
        !jd_check_color(pixel_type, options, nv, color_ops, g_err, (int)sizeof(g_err)))
        return nullptr;
    std::vector<int32_t> one_each;   /* views NULL: one view per file, the same batch as views of ones */
    if (!views) { one_each.assign((size_t)n, 1); views = one_each.data(); }
    JPEGB200_BATCH *b = new (std::nothrow) JPEGB200_BATCH();
    if (!b) return nullptr;
    CreatePlan P;
    P.datas = datas; P.sizes = sizes; P.views = views; P.rois = rois; P.orients = orients; P.out_sizes = out_sizes; P.spec = spec;
    P.draft = draft; P.boxes = boxes; P.gaps = reducing_gaps; P.color = color_ops; P.warp = color_ops ? warp_args : nullptr;
    P.srects.assign(4 * (size_t)nv, 0); P.vok.assign((size_t)nv, 0);
    P.ks.assign(orients ? (size_t)nv : 0u, 0);
    if (options & JPEGB200_OPT_PROGRESSIVE) { P.fscans.resize(JD_PROG_MAX_SCANS); P.ftabs.resize(JD_PROG_MAX_TABS); }
    if (windows) {
        P.windows = windows;
        P.caller_rois = rois;
        P.wn_rois.assign(4 * (size_t)nv, 0);
        P.rois = P.wn_rois.data();
        if (!out_sizes) { P.wn_sizes.assign(2 * (size_t)nv, 1); P.out_sizes = P.wn_sizes.data(); }
    }
    init_batch(b, ctx, P, n, (int)nv, pixel_type, options, rs_filter);
    if (!layout_input(b) || !plan_files(b, P)) { delete b; return nullptr; }
    sort_prog_waves(b);
    build_work_list(b);
    return b;
}

extern "C" void JPEGB200_batchDestroy(JPEGB200_BATCH *b)
{
    if (!b) return;
    cudaSetDevice(b->ctx->device);
    if (b->ss.stream) cudaStreamSynchronize(b->ss.stream);
    if (b->ss.complete()) b->ctx->free_streams.push_back(b->ss);   /* back to the context for the next job */
    else b->ss.destroy();
    if (b->descs_dl) b->ctx->pinpool.put(b->descs_dl, b->descs_dl_bytes);
    delete b;   /* after the synchronise: its device buffers go back to the pool for the next job to reuse */
}

extern "C" int JPEGB200_batchCount(JPEGB200_BATCH *b) { return b ? b->n : 0; }

extern "C" int JPEGB200_batchImageInfo(JPEGB200_BATCH *b, int i, int32_t *width, int32_t *height, int32_t *subsample,
                                       int32_t *out_w, int32_t *out_h, int32_t *status)
{
    if (!b || i < 0 || i >= b->n) return 0;
    const JDInfo &inf = b->infos[b->vfile[i]];
    if (width) *width = inf.width;
    if (height) *height = inf.height;
    if (subsample) *subsample = inf.subsample;
    if (out_w) *out_w = (int32_t)b->descs[i].out_w;
    if (out_h) *out_h = (int32_t)b->descs[i].out_h;
    if (status) *status = b->parse_status[i];
    return 1;
}

extern "C" int64_t JPEGB200_batchOutputBytes(JPEGB200_BATCH *b, int i, int64_t *pitch_bytes)
{
    if (!b || i < 0 || i >= b->n) return 0;
    if (pitch_bytes) *pitch_bytes = (int64_t)b->descs[i].out_pitch;
    return (int64_t)b->descs[i].out_pitch * b->descs[i].out_h * (b->tensor ? b->tn_planes : 1);
}

extern "C" int JPEGB200_batchSetOutputTensor(JPEGB200_BATCH *b, int i, void *out, int64_t pitch, int64_t plane_stride)
{
    if (!b || i < 0 || i >= b->n) return 0;
    if (!b->tensor) { snprintf(g_err, sizeof(g_err), "batchSetOutputTensor on a batch created without a tensor spec"); return 0; }
    if (!jd_check_tensor_output(b->index_base + i, b->tn_elt, (int64_t)b->descs[i].out_pitch, (int64_t)b->descs[i].out_h,
                                b->tn_spec.layout == JPEGB200_LAYOUT_CHW, out, pitch, plane_stride, g_err, (int)sizeof(g_err)))
        return 0;   /* nothing changes */
    b->outs[i] = out;
    b->pitches[i] = pitch > 0 ? pitch : (int64_t)b->descs[i].out_pitch;
    b->tn_plane[i] = plane_stride;
    return 1;
}

extern "C" int JPEGB200_batchSetOutput(JPEGB200_BATCH *b, int i, void *out, int64_t pitch_bytes)
{
    if (!b || i < 0 || i >= b->n) return 0;
    if (b->tensor) return JPEGB200_batchSetOutputTensor(b, i, out, pitch_bytes, 0);
    if (!jd_check_output(b->index_base + i, b->pixel_type, (int64_t)b->descs[i].out_pitch, out, pitch_bytes, 0, g_err, (int)sizeof(g_err)))
        return 0;   /* nothing changes: the image keeps its previous destination and pitch */
    b->outs[i] = out;
    if (pitch_bytes > 0) b->pitches[i] = pitch_bytes;
    return 1;
}

static int batch_stream(JPEGB200_BATCH *b)
{
    CK(cudaSetDevice(b->ctx->device));
    if (!b->ss.stream && !b->ctx->free_streams.empty()) {
        b->ss = b->ctx->free_streams.back();
        b->ctx->free_streams.pop_back();
    }
    if (!b->ss.stream) CK(cudaStreamCreateWithFlags(&b->ss.stream, cudaStreamNonBlocking));
    for (auto &e : b->ss.ev) if (!e) CK(cudaEventCreate(&e));
    return 1;
}

extern "C" void *JPEGB200_batchStream(JPEGB200_BATCH *b) { if (!b || !batch_stream(b)) return nullptr; return (void *)b->ss.stream; }

extern "C" int JPEGB200_batchAllocDeviceOutput(JPEGB200_BATCH *b)
{
    if (!b) return 0;
    CK(cudaSetDevice(b->ctx->device));
    CK(b->d_out.alloc(&b->ctx->pool, b->out_total + 256));
    b->arena_owned = true;
    return 1;
}

extern "C" int JPEGB200_batchGetDeviceOutput(JPEGB200_BATCH *b, int i, void **devptr, int64_t *pitch_bytes)
{
    if (!b || i < 0 || i >= b->n || !b->d_out.p) return 0;
    if (devptr) *devptr = b->d_out.p + b->arena_off[i];
    if (pitch_bytes) *pitch_bytes = (int64_t)b->descs[i].out_pitch;
    return 1;
}

/* synchronous copy of image i's pixels out of the device arena (tests / spot checks) */
extern "C" int JPEGB200_batchReadOutput(JPEGB200_BATCH *b, int i, void *host_dst)
{
    if (!b || i < 0 || i >= b->n || !b->d_out.p || !host_dst) return 0;
    CK(cudaSetDevice(b->ctx->device));
    if (b->ss.stream) CK(cudaStreamSynchronize(b->ss.stream));
    CK(cudaMemcpy(host_dst, b->d_out.p + b->arena_off[i], (size_t)JPEGB200_batchOutputBytes(b, i, nullptr), cudaMemcpyDeviceToHost));
    return 1;
}

extern "C" int JPEGB200_batchUpload(JPEGB200_BATCH *b)
{
    if (!b) return 0;
    if (!batch_stream(b)) return 0;
    const int n = b->n, nf = b->nf;
    CK(b->d_comp.alloc(&b->ctx->pool, b->comp_total + 256));
    CK(b->d_descs.alloc(&b->ctx->pool, n));
    CK(b->d_fdescs.alloc(&b->ctx->pool, nf));
    CK(b->d_quant.alloc(&b->ctx->pool, (size_t)n * 192));
    CK(b->d_luts.alloc(&b->ctx->pool, b->luts.size() ? b->luts.size() : 1));
    CK(b->d_work.alloc(&b->ctx->pool, b->work.size() ? b->work.size() : 1));
    CK(b->d_cta_lut.alloc(&b->ctx->pool, b->cta_lut.size() ? b->cta_lut.size() : 1));
    CK(b->d_seg_img.alloc(&b->ctx->pool, b->seg_img.size()));
    const size_t ns = b->nseg ? b->nseg : 1;
    CK(b->d_seg_start.alloc(&b->ctx->pool, ns + 1)); CK(b->d_seg_jmap.alloc(&b->ctx->pool, ns)); CK(b->d_seg_status.alloc(&b->ctx->pool, ns));
    CK(b->d_seg_nrec.alloc(&b->ctx->pool, ns)); CK(b->d_seg_phase.alloc(&b->ctx->pool, ns + b->nchunks));
    if (b->nchunks) {
        const size_t nc = b->nchunks;
        CK(b->d_filt.alloc(&b->ctx->pool, b->comp_total + 512));
        CK(b->d_cimg_list.alloc(&b->ctx->pool, b->cimg_list.size())); CK(b->d_flen.alloc(&b->ctx->pool, nf));
        CK(b->d_E0.alloc(&b->ctx->pool, nc + 1)); CK(b->d_E1.alloc(&b->ctx->pool, nc + 1)); CK(b->d_Ep.alloc(&b->ctx->pool, nc)); CK(b->d_cfirst.alloc(&b->ctx->pool, nc)); CK(b->d_cn.alloc(&b->ctx->pool, nc)); CK(b->d_cpre.alloc(&b->ctx->pool, nc)); CK(b->d_cjmap.alloc(&b->ctx->pool, nc));
        CK(b->d_cstatus.alloc(&b->ctx->pool, nc)); CK(b->d_cnown.alloc(&b->ctx->pool, nc)); CK(b->d_cdcs.alloc(&b->ctx->pool, 3 * nc)); CK(b->d_cpe.alloc(&b->ctx->pool, 3 * nc));
    }
    CK(b->d_counters.alloc(&b->ctx->pool, 8));
    CK(b->d_blk_hdr.alloc(&b->ctx->pool, b->nblk ? b->nblk : 1));
    CK(b->d_rec.alloc(&b->ctx->pool, b->rec_total + 1024));
    CK(b->d_events.alloc(&b->ctx->pool, JD_EVENT_CAP));
    cudaStream_t st = b->ss.stream;
    CK(cudaEventRecord(b->ss.ev[0], st));
    /* zero the tail padding so word loads past the last file read zeros */
    CK(cudaMemsetAsync(b->d_comp.p + b->comp_total, 0, 256, st));
    if (b->contiguous_in) {
        CK(cudaMemcpyAsync(b->d_comp.p, b->datas[0], b->comp_total, cudaMemcpyHostToDevice, st));
    } else {
        for (int i = 0; i < nf; i++)
            CK(cudaMemcpyAsync(b->d_comp.p + b->comp_off[i], b->datas[i], (size_t)b->sizes[i], cudaMemcpyHostToDevice, st));
    }
    /* the entropy-facing descriptors, once: the kernels rewrite only their status and err_mcu, on every decode.  View
     * descriptors go up with their output placement in batchDecode. */
    CK(cudaMemcpyAsync(b->d_fdescs.p, b->fdescs.data(), sizeof(JDImageDesc) * nf, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b->d_quant.p, b->quant.data(), sizeof(int32_t) * 192 * n, cudaMemcpyHostToDevice, st));
    if (b->luts.size()) CK(cudaMemcpyAsync(b->d_luts.p, b->luts.data(), b->luts.size() * 2, cudaMemcpyHostToDevice, st));
    if (b->work.size()) CK(cudaMemcpyAsync(b->d_work.p, b->work.data(), b->work.size() * 4, cudaMemcpyHostToDevice, st));
    if (b->cta_lut.size()) CK(cudaMemcpyAsync(b->d_cta_lut.p, b->cta_lut.data(), b->cta_lut.size() * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b->d_seg_img.p, b->seg_img.data(), b->seg_img.size() * 4, cudaMemcpyHostToDevice, st));
    if (b->nchunks) {
        CK(cudaMemcpyAsync(b->d_cimg_list.p, b->cimg_list.data(), b->cimg_list.size() * 4, cudaMemcpyHostToDevice, st));
    }
    size_t prog_bytes = 0;
    if (!b->pfiles.empty()) {
        CK(b->d_pscans.alloc(&b->ctx->pool, b->pscans.size()));
        CK(b->d_ptabs.alloc(&b->ctx->pool, b->ptabs.size() ? b->ptabs.size() : 1));
        CK(b->d_pfiles.alloc(&b->ctx->pool, b->pfiles.size()));
        CK(b->d_pplanes.alloc(&b->ctx->pool, nf));
        CK(b->d_perr.alloc(&b->ctx->pool, nf));
        CK(cudaMemcpyAsync(b->d_pscans.p, b->pscans.data(), b->pscans.size() * sizeof(JDProgScan), cudaMemcpyHostToDevice, st));
        if (b->ptabs.size()) CK(cudaMemcpyAsync(b->d_ptabs.p, b->ptabs.data(), b->ptabs.size() * sizeof(JDProgHuff), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(b->d_pfiles.p, b->pfiles.data(), b->pfiles.size() * sizeof(JDProgFile), cudaMemcpyHostToDevice, st));
        prog_bytes = b->pscans.size() * sizeof(JDProgScan) + b->ptabs.size() * sizeof(JDProgHuff) + b->pfiles.size() * sizeof(JDProgFile);
    }
    CK(cudaEventRecord(b->ss.ev[1], st));
    b->uploaded = true;
    b->counters[JPEGB200_C_H2D_BYTES] = (int64_t)(b->comp_total + sizeof(JDImageDesc) * nf + 768 * (size_t)n + b->luts.size() * 2 +
                                                  b->work.size() * 4 + b->cta_lut.size() * 4 + b->seg_img.size() * 4 + prog_bytes);
    return 1;
}

/* ---- IDCT kernel dispatch ---- */
template <int HS, int VS, int NC, int MPB, int PT>
static void launch_idct_pt(const JDIdctArgs &a, dim3 grid, int arith, bool half, cudaStream_t st)
{
    using G = JDGeo<HS, VS, NC, MPB>;
    if (a.roi > 1u) {
        /* oriented stores: one instantiation per transform class */
#define JD_COLOR_ORC(ARITH_, HALF_)                                                                                            \
        if (a.roi == 1u + JD_ORC_FLIP) jdk_idct_color<HS, VS, NC, MPB, PT, ARITH_, HALF_, true, JD_ORC_FLIP><<<grid, G::THREADS, 0, st>>>(a); \
        else jdk_idct_color<HS, VS, NC, MPB, PT, ARITH_, HALF_, true, JD_ORC_TRANSPOSE><<<grid, G::THREADS, 0, st>>>(a);
        if (arith == JPEG_ARITH_SSE2) { if (half) { JD_COLOR_ORC(JPEG_ARITH_SSE2, true) } else { JD_COLOR_ORC(JPEG_ARITH_SSE2, false) } }
        else { if (half) { JD_COLOR_ORC(JPEG_ARITH_SCALAR, true) } else { JD_COLOR_ORC(JPEG_ARITH_SCALAR, false) } }
#undef JD_COLOR_ORC
    } else if (a.roi) {
        if (arith == JPEG_ARITH_SSE2) {
            if (half) jdk_idct_color<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, true, true><<<grid, G::THREADS, 0, st>>>(a);
            else jdk_idct_color<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, false, true><<<grid, G::THREADS, 0, st>>>(a);
        } else {
            if (half) jdk_idct_color<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, true, true><<<grid, G::THREADS, 0, st>>>(a);
            else jdk_idct_color<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, false, true><<<grid, G::THREADS, 0, st>>>(a);
        }
    } else if (arith == JPEG_ARITH_SSE2) {
        if (half) jdk_idct_color<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, true, false><<<grid, G::THREADS, 0, st>>>(a);
        else jdk_idct_color<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, false, false><<<grid, G::THREADS, 0, st>>>(a);
    } else {
        if (half) jdk_idct_color<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, true, false><<<grid, G::THREADS, 0, st>>>(a);
        else jdk_idct_color<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, false, false><<<grid, G::THREADS, 0, st>>>(a);
    }
}

/* Which IDCT kernels a context's decodes take.  JPEGDEC_B200_IDCT (A/B and test switch): unset = the default choice
 * (launch_idct); "lanes" = the 8-lanes-per-block kernels everywhere; "tb" = those, and jdk_idct_tb for 4:2:0 colour at full
 * size, also for the SSE2-build arithmetic; "packed" = the packed kernel for 4:2:0 colour at full size too.
 * JPEGDEC_B200_TB_MPB=16|20 (development switch): force jdk_idct_tb's strip width. */
enum JDIdctKernels { JD_IDCT_DEFAULT, JD_IDCT_LANES, JD_IDCT_TB, JD_IDCT_PACKED };
struct JDIdctChoice { JDIdctKernels kernels; int tb_mpb; };
static const JDIdctChoice &idct_choice()
{
    static const JDIdctChoice choice = [] {
        const char *e = getenv("JPEGDEC_B200_IDCT"), *m = getenv("JPEGDEC_B200_TB_MPB");
        const JDIdctKernels k = !e ? JD_IDCT_DEFAULT : strcmp(e, "lanes") == 0 ? JD_IDCT_LANES : strcmp(e, "tb") == 0 ? JD_IDCT_TB
                                : strcmp(e, "packed") == 0 ? JD_IDCT_PACKED : JD_IDCT_DEFAULT;
        return JDIdctChoice{k, m ? atoi(m) : 0};
    }();
    return choice;
}

template <int HS, int VS, int NC, int MPB, int PT>
static void launch_idct_tb(const JDIdctArgs &a, uint32_t mcus_x, uint32_t mcus_y, uint32_t nimg, int arith, cudaStream_t st)
{
    using G = JDGeoTB<HS, VS, NC, MPB>;
    dim3 grid((mcus_x + MPB - 1) / MPB, mcus_y, nimg);
    static bool carveout_set = false;   /* 10 CTAs of ~17-21 KB static shared memory per SM need the large carveout */
    if (!carveout_set) {
        cudaFuncSetAttribute(jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, true, JD_ORC_FLIP>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, true, JD_ORC_FLIP>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, true, JD_ORC_TRANSPOSE>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, true, JD_ORC_TRANSPOSE>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        carveout_set = true;
    }
    if (a.roi == 1u + JD_ORC_FLIP) {
        if (arith == JPEG_ARITH_SSE2) jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, true, JD_ORC_FLIP><<<grid, G::THREADS, 0, st>>>(a);
        else jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, true, JD_ORC_FLIP><<<grid, G::THREADS, 0, st>>>(a);
    } else if (a.roi == 1u + JD_ORC_TRANSPOSE) {
        if (arith == JPEG_ARITH_SSE2) jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, true, JD_ORC_TRANSPOSE><<<grid, G::THREADS, 0, st>>>(a);
        else jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, true, JD_ORC_TRANSPOSE><<<grid, G::THREADS, 0, st>>>(a);
    } else if (a.roi) {
        if (arith == JPEG_ARITH_SSE2) jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, true><<<grid, G::THREADS, 0, st>>>(a);
        else jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, true><<<grid, G::THREADS, 0, st>>>(a);
    } else if (arith == JPEG_ARITH_SSE2) jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SSE2, false><<<grid, G::THREADS, 0, st>>>(a);
    else jdk_idct_tb<HS, VS, NC, MPB, PT, JPEG_ARITH_SCALAR, false><<<grid, G::THREADS, 0, st>>>(a);
}

/* SSE2-build arithmetic: the packed thread-per-block kernel for every sampling / pixel type, full and half size */
template <int HS, int VS, int NC, int MPB, int PT>
static void launch_idct_p(const JDIdctArgs &a, uint32_t mcus_x, uint32_t mcus_y, uint32_t nimg, bool half, cudaStream_t st)
{
    dim3 grid((mcus_x + MPB - 1) / MPB, mcus_y, nimg);
    static bool carveout_set = false;   /* 7-8 CTAs of ~27 KB static shared memory per SM need the large carveout */
    if (!carveout_set) {
        cudaFuncSetAttribute(jdk_idct_p<HS, VS, NC, MPB, PT, false, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_p<HS, VS, NC, MPB, PT, true, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_p<HS, VS, NC, MPB, PT, false, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_p<HS, VS, NC, MPB, PT, true, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_p<HS, VS, NC, MPB, PT, false, true, JD_ORC_FLIP>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_p<HS, VS, NC, MPB, PT, true, true, JD_ORC_FLIP>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_p<HS, VS, NC, MPB, PT, false, true, JD_ORC_TRANSPOSE>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(jdk_idct_p<HS, VS, NC, MPB, PT, true, true, JD_ORC_TRANSPOSE>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        carveout_set = true;
    }
    if (a.roi == 1u + JD_ORC_FLIP) {
        if (half) jdk_idct_p<HS, VS, NC, MPB, PT, true, true, JD_ORC_FLIP><<<grid, 128, 0, st>>>(a);
        else jdk_idct_p<HS, VS, NC, MPB, PT, false, true, JD_ORC_FLIP><<<grid, 128, 0, st>>>(a);
    } else if (a.roi == 1u + JD_ORC_TRANSPOSE) {
        if (half) jdk_idct_p<HS, VS, NC, MPB, PT, true, true, JD_ORC_TRANSPOSE><<<grid, 128, 0, st>>>(a);
        else jdk_idct_p<HS, VS, NC, MPB, PT, false, true, JD_ORC_TRANSPOSE><<<grid, 128, 0, st>>>(a);
    } else if (a.roi) {
        if (half) jdk_idct_p<HS, VS, NC, MPB, PT, true, true><<<grid, 128, 0, st>>>(a);
        else jdk_idct_p<HS, VS, NC, MPB, PT, false, true><<<grid, 128, 0, st>>>(a);
    } else if (half) jdk_idct_p<HS, VS, NC, MPB, PT, true, false><<<grid, 128, 0, st>>>(a);
    else jdk_idct_p<HS, VS, NC, MPB, PT, false, false><<<grid, 128, 0, st>>>(a);
}

template <int HS, int VS>
static int launch_idct_packed(const JDIdctArgs &a, uint32_t mcus_x, uint32_t mcus_y, uint32_t nimg, int ncomp, int ptclass, bool half, cudaStream_t st)
{
    constexpr int MPB1 = 128 / (HS * VS);            /* luma only: HS * VS blocks per MCU */
    constexpr int MPB3 = (HS * VS == 4) ? 20 : (HS * VS == 2) ? 30 : 40;
    if (ptclass == JD_PT_GRAY) { launch_idct_p<HS, VS, 1, MPB1, JD_PT_GRAY>(a, mcus_x, mcus_y, nimg, half, st); return 1; }
    if (ncomp == 1) {
        if (HS != 1 || VS != 1 || ptclass != JD_PT_565) return 0;
        launch_idct_p<1, 1, 1, 128, JD_PT_565>(a, mcus_x, mcus_y, nimg, half, st);
        return 1;
    }
    if (HS == 2 && VS == 2) {
        /* strips of 20 MCUs (320 px) unless strips of 16 waste fewer MCU slots (1920 and 3840 px divide evenly by 320) */
        const uint32_t pad16 = (mcus_x + 15) / 16 * 16 - mcus_x, pad20 = (mcus_x + 19) / 20 * 20 - mcus_x;
        if (pad20 <= pad16) {
            if (ptclass == JD_PT_565) launch_idct_p<2, 2, 3, 20, JD_PT_565>(a, mcus_x, mcus_y, nimg, half, st);
            else launch_idct_p<2, 2, 3, 20, JD_PT_8888>(a, mcus_x, mcus_y, nimg, half, st);
        } else {
            if (ptclass == JD_PT_565) launch_idct_p<2, 2, 3, 16, JD_PT_565>(a, mcus_x, mcus_y, nimg, half, st);
            else launch_idct_p<2, 2, 3, 16, JD_PT_8888>(a, mcus_x, mcus_y, nimg, half, st);
        }
        return 1;
    }
    if (ptclass == JD_PT_565) launch_idct_p<HS, VS, 3, MPB3, JD_PT_565>(a, mcus_x, mcus_y, nimg, half, st);
    else launch_idct_p<HS, VS, 3, MPB3, JD_PT_8888>(a, mcus_x, mcus_y, nimg, half, st);
    return 1;
}

template <int HS, int VS, int MPB3, int MPB1>
static int launch_idct_geo(const JDIdctArgs &a, uint32_t mcus_x, uint32_t mcus_y, uint32_t nimg, int ncomp, int ptclass,
                           int arith, bool half, cudaStream_t st)
{
    const JDIdctChoice &choice = idct_choice();
    if (choice.kernels != JD_IDCT_LANES && !half && HS == 2 && VS == 2 && ncomp == 3 && ptclass != JD_PT_GRAY) {
        /* 4:2:0 colour, full size: the throughput configuration */
        /* strips of 20 MCUs (320 px) unless that wastes more MCU slots than strips of 16 (1920 and 3840 px divide evenly by 320;
         * measured faster there than strips of 16) */
        const uint32_t pad16 = (mcus_x + 15) / 16 * 16 - mcus_x, pad20 = (mcus_x + 19) / 20 * 20 - mcus_x;
        const bool wide = choice.tb_mpb == 20 || (choice.tb_mpb == 0 && pad20 <= pad16);
        if (wide) {
            if (ptclass == JD_PT_565) launch_idct_tb<2, 2, 3, 20, JD_PT_565>(a, mcus_x, mcus_y, nimg, arith, st);
            else launch_idct_tb<2, 2, 3, 20, JD_PT_8888>(a, mcus_x, mcus_y, nimg, arith, st);
        } else {
            if (ptclass == JD_PT_565) launch_idct_tb<2, 2, 3, 16, JD_PT_565>(a, mcus_x, mcus_y, nimg, arith, st);
            else launch_idct_tb<2, 2, 3, 16, JD_PT_8888>(a, mcus_x, mcus_y, nimg, arith, st);
        }
        return 1;
    }
    if (ptclass == JD_PT_GRAY) {
        dim3 grid((mcus_x + MPB1 - 1) / MPB1, mcus_y, nimg);
        launch_idct_pt<HS, VS, 1, MPB1, JD_PT_GRAY>(a, grid, arith, half, st);
    } else if (ncomp == 1) {
        if (HS != 1 || VS != 1 || ptclass != JD_PT_565) return 0;
        dim3 grid((mcus_x + MPB1 - 1) / MPB1, mcus_y, nimg);
        launch_idct_pt<1, 1, 1, MPB1, JD_PT_565>(a, grid, arith, half, st);
    } else {
        dim3 grid((mcus_x + MPB3 - 1) / MPB3, mcus_y, nimg);
        if (ptclass == JD_PT_565) launch_idct_pt<HS, VS, 3, MPB3, JD_PT_565>(a, grid, arith, half, st);
        else launch_idct_pt<HS, VS, 3, MPB3, JD_PT_8888>(a, grid, arith, half, st);
    }
    return 1;
}

/* One IDCT + colour launch for a run of nimg images of one sampling.  The SSE2-build arithmetic takes the packed
 * thread-per-block kernel for every sampling / pixel type / half scale except 4:2:0 colour at full size, which keeps
 * jdk_idct_tb (measured faster there -- there is no packed 16-bit subtract instruction, __vsub2 costs three, which eats what
 * the packed adds save).  0 when there is no kernel for the combination. */
static int launch_idct(const JDIdctArgs &ia, int subsample, int ncomp, int ptclass, int arith, bool half, uint32_t mcus_x,
                       uint32_t mcus_y, uint32_t nimg, cudaStream_t st)
{
    const JDIdctKernels k = idct_choice().kernels;
    const bool tb_case = subsample == 0x22 && ncomp == 3 && ptclass != JD_PT_GRAY && !half;
    const bool packed = arith == JPEG_ARITH_SSE2 && k != JD_IDCT_LANES && k != JD_IDCT_TB && (!tb_case || k == JD_IDCT_PACKED);
#define JD_IDCT_SAMPLING(HS_, VS_, MPB3_, MPB1_)                                                                 \
    return packed ? launch_idct_packed<HS_, VS_>(ia, mcus_x, mcus_y, nimg, ncomp, ptclass, half, st)             \
                  : launch_idct_geo<HS_, VS_, MPB3_, MPB1_>(ia, mcus_x, mcus_y, nimg, ncomp, ptclass, arith, half, st)
    switch (subsample) {
        case 0x00: case 0x11: JD_IDCT_SAMPLING(1, 1, 16, 32);
        case 0x21: JD_IDCT_SAMPLING(2, 1, 8, 16);
        case 0x12: JD_IDCT_SAMPLING(1, 2, 8, 16);
        case 0x22: JD_IDCT_SAMPLING(2, 2, 8, 8);
    }
#undef JD_IDCT_SAMPLING
    return 0;
}

/* ---- JPEGB200_batchDecode, step by step.  What several steps share lives on its stack. ---- */
struct DecodeState {
    std::vector<JDImageDesc> descs_stage;   /* the descriptors the kernels read: b->descs keeps the tight pitch (JPEGB200_batchOutputBytes, the arena) */
    bool user_dev_out = false;              /* the pixels go to the caller's device pointers, not to the arena */
    uint8_t *out_base = nullptr;            /* the destination: the arena, or the lowest of the caller's pointers */
    uint8_t *pipe_out = nullptr;            /* where the pixel pipeline (IDCT, resize) writes: out_base, or the tensor staging */
    uint8_t *stage_out = nullptr;           /* where the IDCT stage writes: pipe_out, or the gray stage / the resize source */
    uint32_t tn_ctas = 0, rs_ctas[4] = {0u, 0u, 0u, 0u};
    uint32_t bx_ctas[2] = {0u, 0u};         /* box batches: jdk_resize_coeffs_box, jdk_reduce */
    std::vector<uint32_t> co_ctas;          /* colour operations: CTAs of each jdk_color launch */
    std::vector<uint32_t> bl_first;         /* blurs: the first bl_desc entry of each cut index (one past the last at nl) */
    std::vector<uint32_t> bl_ctas;          /* CTAs of each cut index's jdk_blur pair: horizontal, vertical */
    std::vector<uint32_t> au_first;         /* sharpness and geometric ops: the first au_desc entry of each cut index */
    std::vector<uint32_t> au_ctas;          /* CTAs of each cut index's jdk_augment_copy (jdk_augment's, then jdk_augment_rs's) */
    std::vector<uint32_t> au_nn;            /* per cut index: the entries and CTAs of jdk_augment, then those of jdk_augment
                                               and jdk_augment_rs together (the rest warp) */
    std::vector<uint32_t> jq_first;         /* JPEG ops: the first jq_desc entry of each cut index (one past the last at nl) */
    std::vector<uint32_t> jq_ctas;          /* CTAs of each cut index's jdk_jq_fwd, then of its jdk_jq_color */
    std::vector<uint8_t> co_lut;            /* per cut index: some view posterizes, inverts, applies a LUT or counts a
                                               histogram there (jdk_color_lut) */
    unsigned long long *co_hist = nullptr;  /* the histogram slots */
    uint32_t co_nsum = 0;                   /* sum slots per view: the most cuts (contrasts and blurs) of any view */
    int launches = 0;
};

/* coefficient planes of the progressive files, one pooled buffer each: a file whose plane the device cannot hold gets
 * JPEG_ERROR_MEMORY (all of its views) and the others decode.  Writes d_pplane, pplane_ptr, pwalkers, parse_status. */
static int alloc_prog_planes(JPEGB200_BATCH *b)
{
    if (b->pfiles.empty()) return 1;
    cudaStream_t st = b->ss.stream;
    b->d_pplane.resize(b->nf);
    b->pplane_ptr.assign(b->nf, nullptr);
    b->pwalkers = 0;
    for (const JDProgFile &pf : b->pfiles) {
        const int f = (int)pf.file;
        if (b->d_pplane[f].alloc(&b->ctx->pool, (size_t)b->pplane[f] / 2) != cudaSuccess) {
            cudaGetLastError();
            for (int i = 0; i < b->n; i++) if (b->vfile[i] == f) b->parse_status[i] = JPEG_ERROR_MEMORY;
            continue;
        }
        b->pplane_ptr[f] = b->d_pplane[f].p;
        CK(cudaMemsetAsync(b->pplane_ptr[f], 0, (size_t)b->pplane[f], st));
    }
    for (const JDProgScan &s : b->pscans) if (b->pplane_ptr[s.img]) b->pwalkers++;
    CK(cudaMemcpyAsync(b->d_pplanes.p, b->pplane_ptr.data(), sizeof(int16_t *) * b->nf, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(b->d_perr.p, 0xFF, sizeof(uint32_t) * b->nf, st));
    return 1;
}

/* output placement: the caller's device pointers (checked before anything is enqueued) or the arena.  Writes
 * D.user_dev_out, D.out_base and D.descs_stage with each image's out_off / out_pitch. */
static int place_outputs(JPEGB200_BATCH *b, DecodeState &D)
{
    const int n = b->n;
    if (b->out_device && !b->arena_owned) {
        D.user_dev_out = true;
        for (int i = 0; i < n; i++) if (!b->outs[i] && b->parse_status[i] == JPEG_SUCCESS) D.user_dev_out = false;
        bool any_ptr = false;
        for (int i = 0; i < n; i++) if (b->outs[i]) any_ptr = true;
        if (!D.user_dev_out && any_ptr) { snprintf(g_err, sizeof(g_err), "device output pointers given for some images only"); return 0; }
        /* the kernels store through these pointers: refuse misaligned ones before anything is enqueued */
        for (int i = 0; i < n; i++)
            if (b->outs[i] && !b->tensor && !jd_check_output(b->index_base + i, b->pixel_type, (int64_t)b->descs[i].out_pitch, b->outs[i], b->pitches[i], 1,
                                                             g_err, (int)sizeof(g_err)))
                return 0;
        for (int i = 0; i < n && b->tensor; i++) {
            /* the kernel stores through these pointers: they must be device memory of this context's GPU */
            if (!b->outs[i]) continue;
            cudaPointerAttributes pa;
            const cudaError_t e = cudaPointerGetAttributes(&pa, b->outs[i]);
            if (e != cudaSuccess) cudaGetLastError();
            if (e != cudaSuccess || (pa.type != cudaMemoryTypeDevice && pa.type != cudaMemoryTypeManaged) || pa.device != b->ctx->device) {
                snprintf(g_err, sizeof(g_err), "tensor output of image %d: %p is not device memory of GPU %d", b->index_base + i,
                         b->outs[i], b->ctx->device);
                return 0;
            }
        }
    }
    D.descs_stage = b->descs;
    if (D.user_dev_out) {
        /* user device pointers: offsets relative to the lowest pointer */
        uintptr_t lo = ~(uintptr_t)0;
        for (int i = 0; i < n; i++) if (b->outs[i] && (uintptr_t)b->outs[i] < lo) lo = (uintptr_t)b->outs[i];
        D.out_base = (uint8_t *)lo;
        for (int i = 0; i < n; i++) {
            D.descs_stage[i].out_off = b->outs[i] ? (uint64_t)((uintptr_t)b->outs[i] - lo) : 0;
            D.descs_stage[i].out_pitch = (uint32_t)b->pitches[i];
        }
    } else {
        if (!b->d_out.p) { CK(b->d_out.alloc(&b->ctx->pool, b->out_total + 256)); b->arena_owned = true; }
        D.out_base = b->d_out.p;
        for (int i = 0; i < n; i++) D.descs_stage[i].out_off = b->arena_off[i];
    }
    D.pipe_out = D.out_base;
    return 1;
}

/* tensor: the pipeline writes U tightly into d_tn (D.pipe_out) where it would have written the destination; jdk_tensor then
 * writes the destination.  Uploads tn_desc and the element table; rewrites D.descs_stage for the stage before it. */
static int stage_tensor(JPEGB200_BATCH *b, DecodeState &D)
{
    const int n = b->n;
    cudaStream_t st = b->ss.stream;
    b->tn_desc.assign(n, JDTensorDesc{});
    constexpr uint32_t px_per_thread[5] = {0u, 16u, 8u, 0u, 4u};
    const uint32_t PX = px_per_thread[b->tn_elt];
    uint64_t so = 0, ctas = 0;
    for (int i = 0; i < n; i++) {
        JDTensorDesc &t = b->tn_desc[i];
        t.blk = (uint32_t)ctas;
        if (b->parse_status[i] != JPEG_SUCCESS) continue;
        const JDImageDesc &d = b->descs[i];
        t.w = d.out_w; t.h = d.out_h; t.swap = b->tn_swap[i];
        t.src_off = so;
        so += (uint64_t)b->tn_stage[i];
        t.dst_off = D.descs_stage[i].out_off;
        t.pitch = D.user_dev_out ? (uint64_t)b->pitches[i] : (uint64_t)d.out_pitch;
        t.plane = (D.user_dev_out && b->tn_plane[i]) ? (uint64_t)b->tn_plane[i] : t.pitch * d.out_h;
        ctas += ((uint64_t)(d.out_w + PX - 1) / PX * d.out_h + JD_TN_THREADS - 1) / JD_TN_THREADS;
        D.descs_stage[i].out_off = t.src_off;
        D.descs_stage[i].out_pitch = d.out_w * (uint32_t)b->tn_bpp;
    }
    if (ctas >= (1ull << 31)) { snprintf(g_err, sizeof(g_err), "tensor output: too many elements in one job"); return 0; }
    D.tn_ctas = (uint32_t)ctas;
    CK(b->d_tn.alloc(&b->ctx->pool, so + 256));
    CK(b->d_tn_tab.alloc(&b->ctx->pool, 3 * 256));
    CK(b->d_tn_desc.alloc(&b->ctx->pool, n));
    CK(cudaMemcpyAsync(b->d_tn_tab.p, b->tn_table.data(), 3 * 256 * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b->d_tn_desc.p, b->tn_desc.data(), sizeof(JDTensorDesc) * n, cudaMemcpyHostToDevice, st));
    D.pipe_out = b->d_tn.p;
    return 1;
}

/* colour operations: where each view's final uint8 image lies before the resize and dither stages redirect the stages
 * before them (D.pipe_out + out_off, out_pitch).  Uploads co_desc, the per-launch CTA starts and zeroed contrast sums, and
 * for the blurs bl_desc (the views blurring at each cut index, in cut order) with their CTA starts. */
static int stage_color(JPEGB200_BATCH *b, DecodeState &D)
{
    const int n = b->n;
    cudaStream_t st = b->ss.stream;
    uint32_t nl = 0;
    for (int i = 0; i < n; i++)
        if (b->parse_status[i] == JPEG_SUCCESS && b->co_plans[i].nops && b->co_plans[i].ncontrast + 1 > nl) nl = b->co_plans[i].ncontrast + 1;
    if (nl == 0) return 1;   /* no view has an operation */
    D.co_nsum = nl - 1;
    b->co_desc.assign(n, JDColorDesc{});
    b->co_blk.assign((size_t)nl * n, 0);
    std::vector<uint64_t> ctas(nl, 0);
    D.co_lut.assign(nl, 0);
    std::vector<uint32_t> hslot((size_t)nl * n, 0);
    uint32_t nslots = 0;
    for (int i = 0; i < n; i++) {
        for (uint32_t s = 0; s < nl; s++) b->co_blk[(size_t)s * n + i] = (uint32_t)ctas[s];
        const JDColorPlan &p = b->co_plans[i];
        if (b->parse_status[i] != JPEG_SUCCESS || p.nops == 0) continue;
        JDColorDesc &c = b->co_desc[i];
        c.off = D.descs_stage[i].out_off; c.pitch = D.descs_stage[i].out_pitch;
        c.w = b->descs[i].out_w; c.h = b->descs[i].out_h;
        c.bgr = b->co_bgr[i];
        c.plan = p;
        const uint64_t per = ((uint64_t)c.w * c.h + JD_CO_THREADS - 1) / JD_CO_THREADS;
        for (uint32_t s = 0; s <= p.ncontrast; s++) {
            /* segment s has per-pixel operations after its own-kernel op, or sums L for the contrast after it, or counts
             * the histogram for the autocontrast or equalize after it */
            const uint32_t k0 = p.seg[s] + (p.seg[s] < p.seg[s + 1] && JD_CO_OWN_KERNEL(p.op[p.seg[s]]) ? 1u : 0u);
            const uint32_t next = s < p.ncontrast ? p.op[p.seg[s + 1]] : 0u;
            if (k0 < p.seg[s + 1] || next == JD_CO_CONTRAST || JD_CO_LUT(next)) ctas[s] += per;
            if (JD_CO_LUT(next)) { hslot[(size_t)s * n + i] = nslots++; D.co_lut[s] = 1; }
            for (uint32_t k = p.seg[s]; k < p.seg[s + 1]; k++)
                if (JD_CO_LUT(p.op[k]) || p.op[k] == JD_CO_POSTERIZE || p.op[k] == JD_CO_INVERT) D.co_lut[s] = 1;
        }
    }
    /* blurs: at cut index s, the views whose segment s starts with one */
    b->bl_desc.clear();
    D.bl_first.assign(nl + 1, 0);
    D.bl_ctas.assign(2 * (size_t)nl, 0);
    std::vector<uint32_t> hblk, vblk;
    uint64_t soff = 0;
    std::vector<uint64_t> soffs(n, 0);
    for (int i = 0; i < n; i++) {   /* the scratch copies first, then the histogram slots */
        if (b->parse_status[i] != JPEG_SUCCESS) continue;
        const JDColorPlan &p = b->co_plans[i];
        uint64_t nlut = 0;
        for (uint32_t k = 0; k < p.nops; k++) nlut += JD_CO_LUT(p.op[k]) ? 1u : 0u;
        const uint64_t img = (uint64_t)b->bl_scratch[i] - nlut * JD_AU_HIST * sizeof(unsigned long long);
        if (img) { soffs[i] = soff; soff += img; }
    }
    const uint64_t hbytes = (uint64_t)nslots * JD_AU_HIST * sizeof(unsigned long long);
    for (uint32_t s = 1; s < nl; s++) {
        D.bl_first[s] = (uint32_t)b->bl_desc.size();
        for (int i = 0; i < n; i++) {
            const JDColorPlan &p = b->co_plans[i];
            if (b->parse_status[i] != JPEG_SUCCESS || s > p.ncontrast || p.op[p.seg[s]] != JD_CO_BLUR) continue;
            JDBlurDesc x{};
            x.off = b->co_desc[i].off; x.pitch = b->co_desc[i].pitch; x.soff = soffs[i];
            x.w = b->co_desc[i].w; x.h = b->co_desc[i].h;
            x.k = b->co_blur[i].b[p.seg[s]];
            b->bl_desc.push_back(x);
            hblk.push_back(D.bl_ctas[2 * s]); vblk.push_back(D.bl_ctas[2 * s + 1]);
            D.bl_ctas[2 * s] += (x.h + JD_BL_THREADS / 32 - 1) / (JD_BL_THREADS / 32);   /* 8 rows per CTA */
            D.bl_ctas[2 * s + 1] += (x.w + 31) / 32;                                       /* 32 columns per CTA */
        }
    }
    D.bl_first[nl] = (uint32_t)b->bl_desc.size();
    /* sharpness, geometric and warp ops: at cut index s, the views whose segment s starts with one -- first those that
     * sharpen or move pixels with NEAREST (jdk_augment), then those that resample (jdk_augment_rs), each with its matrix in
     * au_mat, then those that warp (jdk_warp), each with its coefficients and fill in au_warp */
    b->au_desc.clear();
    b->au_mat.clear();
    b->au_warp.clear();
    b->au_tab.clear();
    D.au_first.assign(nl + 1, 0);
    D.au_ctas.assign(nl, 0);
    D.au_nn.assign(4 * (size_t)nl, 0);
    bool any_rs = false, any_warp = false;
    for (uint32_t s = 1; s < nl; s++) {
        D.au_first[s] = (uint32_t)b->au_desc.size();
        for (int rs = 0; rs < 3; rs++) {
            for (int i = 0; i < n; i++) {
                const JDColorPlan &p = b->co_plans[i];
                if (b->parse_status[i] != JPEG_SUCCESS || s > p.ncontrast) continue;
                const uint32_t op = p.op[p.seg[s]];
                if (rs == 2 ? !JD_CO_WARP(op) : rs ? !JD_CO_RESAMPLE(op) || JD_CO_WARP(op) : op != JD_CO_SHARPNESS && !JD_CO_GEOMETRIC(op)) continue;
                JDAugDesc x{};
                x.off = b->co_desc[i].off; x.pitch = b->co_desc[i].pitch; x.soff = soffs[i];
                x.w = b->co_desc[i].w; x.h = b->co_desc[i].h;
                x.op = op; x.arg = p.arg[p.seg[s]];
                x.m = b->co_aug[i].a[p.seg[s]];
                x.blk = D.au_ctas[s];
                const uint64_t c = D.au_ctas[s] + ((uint64_t)x.w * x.h + JD_AU_THREADS - 1) / JD_AU_THREADS;
                if (c >= (1ull << 31)) { snprintf(g_err, sizeof(g_err), "colour operations: too many pixels in one job"); return 0; }
                D.au_ctas[s] = (uint32_t)c;
                b->au_desc.push_back(x);
                JDAugMat mt;
                memcpy(mt.m, b->co_rs[i].mat[p.seg[s]], sizeof(mt.m));
                b->au_mat.push_back(mt);
                JDWarpDesc wd{};
                if (rs == 2) {   /* the fill in the view's byte order, alpha 0xFF */
                    const JDWarpPlan &wp = b->co_warp[i];
                    memcpy(wd.c, wp.c[p.seg[s]], sizeof(wd.c));
                    const uint32_t f = wp.fill[p.seg[s]];
                    wd.fill = b->ptclass == JD_PT_GRAY ? (f & 255u)
                            : b->co_bgr[i] ? (f >> 16 & 255u) | (f & 0xFF00u) | (f & 255u) << 16 | 0xFF000000u : f | 0xFF000000u;
                    if (op == JD_CO_AFFINE && wd.c[1] == 0.0 && wd.c[3] == 0.0) {   /* NEAREST, scale and translate only */
                        wd.tab = (uint32_t)b->au_tab.size();
                        b->au_tab.resize(b->au_tab.size() + x.w + x.h);
                        jd_walk_table(wd.c, x.w, x.h, b->au_tab.data() + wd.tab);
                    }
                }
                b->au_warp.push_back(wd);
                any_rs = any_rs || rs == 1;
                any_warp = any_warp || rs == 2;
            }
            if (rs < 2) { D.au_nn[4 * s + 2 * rs] = (uint32_t)b->au_desc.size() - D.au_first[s]; D.au_nn[4 * s + 2 * rs + 1] = D.au_ctas[s]; }
        }
    }
    D.au_first[nl] = (uint32_t)b->au_desc.size();
    /* JPEG ops: at cut index s, the views whose segment s starts with one; one table pair per distinct quality */
    b->jq_desc.clear();
    b->jq_tab.clear();
    D.jq_first.assign(nl + 1, 0);
    D.jq_ctas.assign(2 * (size_t)nl, 0);
    int32_t tab_of[101];
    for (int q = 0; q <= 100; q++) tab_of[q] = -1;
    for (uint32_t s = 1; s < nl; s++) {
        D.jq_first[s] = (uint32_t)b->jq_desc.size();
        uint64_t cf = 0, cc = 0;
        for (int i = 0; i < n; i++) {
            const JDColorPlan &p = b->co_plans[i];
            if (b->parse_status[i] != JPEG_SUCCESS || s > p.ncontrast || !JD_CO_JQ(p.op[p.seg[s]])) continue;
            const uint32_t q = p.arg[p.seg[s]];
            if (tab_of[q] < 0) {
                tab_of[q] = (int32_t)(b->jq_tab.size() / 128);
                b->jq_tab.resize(b->jq_tab.size() + 128);
                jd_jq_tables((int)q, b->jq_tab.data() + b->jq_tab.size() - 128);
            }
            const bool gray = b->ptclass == JD_PT_GRAY;
            uint32_t hs = 1u, vs = 1u;
            if (!gray) jd_jq_factors(p.op[p.seg[s]], &hs, &vs);
            JDJqDesc x{};
            x.off = b->co_desc[i].off; x.pitch = b->co_desc[i].pitch; x.soff = soffs[i];
            x.g = jd_jq_geo(b->co_desc[i].w, b->co_desc[i].h, hs, vs);
            x.bgr = b->co_bgr[i];
            x.tab = (uint32_t)tab_of[q];
            x.blk = (uint32_t)cf; x.cblk = (uint32_t)cc;
            cf += ((uint64_t)x.g.nmx * x.g.nmy * jd_jq_bpm(hs, vs, gray) + JD_JQ_THREADS - 1) / JD_JQ_THREADS;
            if (!gray) cc += ((uint64_t)x.g.w * x.g.h + JD_CO_THREADS - 1) / JD_CO_THREADS;
            if (cf >= (1ull << 31) || cc >= (1ull << 31)) { snprintf(g_err, sizeof(g_err), "colour operations: too many pixels in one job"); return 0; }
            b->jq_desc.push_back(x);
        }
        D.jq_ctas[2 * s] = (uint32_t)cf; D.jq_ctas[2 * s + 1] = (uint32_t)cc;
    }
    D.jq_first[nl] = (uint32_t)b->jq_desc.size();
    if (!b->jq_desc.empty()) {
        CK(b->d_jq_desc.alloc(&b->ctx->pool, b->jq_desc.size()));
        CK(cudaMemcpyAsync(b->d_jq_desc.p, b->jq_desc.data(), sizeof(JDJqDesc) * b->jq_desc.size(), cudaMemcpyHostToDevice, st));
        CK(b->d_jq_tab.alloc(&b->ctx->pool, b->jq_tab.size()));
        CK(cudaMemcpyAsync(b->d_jq_tab.p, b->jq_tab.data(), sizeof(uint16_t) * b->jq_tab.size(), cudaMemcpyHostToDevice, st));
    }
    if (soff + hbytes) CK(b->d_bl.alloc(&b->ctx->pool, soff + hbytes));
    if (!b->au_desc.empty()) {
        CK(b->d_au_desc.alloc(&b->ctx->pool, b->au_desc.size()));
        CK(cudaMemcpyAsync(b->d_au_desc.p, b->au_desc.data(), sizeof(JDAugDesc) * b->au_desc.size(), cudaMemcpyHostToDevice, st));
    }
    if (any_rs) {
        CK(b->d_au_mat.alloc(&b->ctx->pool, b->au_mat.size()));
        CK(cudaMemcpyAsync(b->d_au_mat.p, b->au_mat.data(), sizeof(JDAugMat) * b->au_mat.size(), cudaMemcpyHostToDevice, st));
    }
    if (any_warp) {
        CK(b->d_au_warp.alloc(&b->ctx->pool, b->au_warp.size()));
        CK(cudaMemcpyAsync(b->d_au_warp.p, b->au_warp.data(), sizeof(JDWarpDesc) * b->au_warp.size(), cudaMemcpyHostToDevice, st));
    }
    if (!b->au_tab.empty()) {
        CK(b->d_au_tab.alloc(&b->ctx->pool, b->au_tab.size()));
        CK(cudaMemcpyAsync(b->d_au_tab.p, b->au_tab.data(), sizeof(int16_t) * b->au_tab.size(), cudaMemcpyHostToDevice, st));
    }
    if (nslots) {   /* soff is 256-byte aligned: the slots are 64-bit aligned */
        D.co_hist = reinterpret_cast<unsigned long long *>(b->d_bl.p + soff);
        CK(cudaMemsetAsync(D.co_hist, 0, hbytes, st));
        CK(b->d_co_hslot.alloc(&b->ctx->pool, (size_t)nl * n));
        CK(cudaMemcpyAsync(b->d_co_hslot.p, hslot.data(), sizeof(uint32_t) * nl * n, cudaMemcpyHostToDevice, st));
    }
    if (!b->bl_desc.empty()) {
        const size_t m = b->bl_desc.size();
        b->bl_blk = hblk;
        b->bl_blk.insert(b->bl_blk.end(), vblk.begin(), vblk.end());
        CK(b->d_bl_desc.alloc(&b->ctx->pool, m));
        CK(b->d_bl_blk.alloc(&b->ctx->pool, 2 * m));
        CK(cudaMemcpyAsync(b->d_bl_desc.p, b->bl_desc.data(), sizeof(JDBlurDesc) * m, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(b->d_bl_blk.p, b->bl_blk.data(), sizeof(uint32_t) * 2 * m, cudaMemcpyHostToDevice, st));
    }
    D.co_ctas.assign(nl, 0);
    for (uint32_t s = 0; s < nl; s++) {
        if (ctas[s] >= (1ull << 31)) { snprintf(g_err, sizeof(g_err), "colour operations: too many pixels in one job"); return 0; }
        D.co_ctas[s] = (uint32_t)ctas[s];
    }
    CK(b->d_co_desc.alloc(&b->ctx->pool, n));
    CK(b->d_co_blk.alloc(&b->ctx->pool, (size_t)nl * n));
    CK(b->d_co_sum.alloc(&b->ctx->pool, D.co_nsum ? (size_t)D.co_nsum * n : 1));
    CK(cudaMemcpyAsync(b->d_co_desc.p, b->co_desc.data(), sizeof(JDColorDesc) * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b->d_co_blk.p, b->co_blk.data(), sizeof(uint32_t) * nl * n, cudaMemcpyHostToDevice, st));
    if (D.co_nsum) CK(cudaMemsetAsync(b->d_co_sum.p, 0, sizeof(unsigned long long) * D.co_nsum * n, st));
    return 1;
}

/* resize: the IDCT stage writes S tightly into d_rs; jdk_resize_v writes where the IDCT would have.  Uploads rs_desc with the
 * CTA prefix sums of the four passes (D.rs_ctas); rewrites D.descs_stage for the IDCT stage. */
static int stage_resize(JPEGB200_BATCH *b, DecodeState &D)
{
    const int n = b->n;
    const int bp = bytes_per_pixel_class(b->ptclass);
    b->rs_desc.assign(n, JDResizeDesc{});
    if (b->box) b->bx_desc.assign(n, JDBoxDesc{});
    uint64_t so = 0, co = 0, ctas[4] = {0, 0, 0, 0}, bx_ctas[2] = {0, 0};
    for (int i = 0; i < n; i++) {
        JDResizeDesc &r = b->rs_desc[i];
        r.blk_c = (uint32_t)ctas[0]; r.blk_h = (uint32_t)ctas[1]; r.blk_v = (uint32_t)ctas[2]; r.blk_h2 = (uint32_t)ctas[3];
        if (b->box) { b->bx_desc[i].blk_c = (uint32_t)bx_ctas[0]; b->bx_desc[i].blk_r = (uint32_t)bx_ctas[1]; }
        if (b->parse_status[i] != JPEG_SUCCESS) continue;
        const JDResizePlan &rp = b->rs_plans[i];
        const uint32_t sw = b->rs_src_w[i], sh = b->rs_src_h[i];   /* S, where the IDCT stage writes */
        r.src_w = sw; r.src_h = sh; r.dst_w = b->descs[i].out_w; r.dst_h = b->descs[i].out_h;
        r.dst_off = D.descs_stage[i].out_off; r.dst_pitch = D.descs_stage[i].out_pitch;
        r.ksize_h = (uint32_t)rp.ksize_h; r.ksize_v = (uint32_t)rp.ksize_v;
        r.ybox0 = (uint32_t)rp.ybox0; r.rows = (uint32_t)rp.rows;
        r.flags = (rp.need_h ? 1u : 0u) | (rp.need_v ? 2u : 0u) | (rp.vfirst ? 4u : 0u);
        r.in_w = sw; r.in_h = sh; r.full_w = r.dst_w; r.full_h = r.dst_h;
        r.wx1 = r.dst_w; r.wy1 = r.dst_h;
        if (b->window) {
            const JDWindowPlan &wp = b->wn_plans[i];
            r.in_w = (uint32_t)b->wn_full[2 * (size_t)i]; r.in_h = (uint32_t)b->wn_full[2 * (size_t)i + 1];
            r.full_w = (uint32_t)b->wn_out[2 * (size_t)i]; r.full_h = (uint32_t)b->wn_out[2 * (size_t)i + 1];
            r.sx = (uint32_t)wp.sx; r.sy = (uint32_t)wp.sy;
            r.wx0 = (uint32_t)wp.x0; r.wx1 = (uint32_t)wp.x1; r.wy0 = (uint32_t)wp.y0; r.wy1 = (uint32_t)wp.y1;
            r.win_x = b->wn_win[4 * (size_t)i]; r.win_y = b->wn_win[4 * (size_t)i + 1];
        }
        r.src_off = so;
        so += align256((size_t)sw * sh * bp);
        if (b->box) {
            /* the resize reads the reduced image (written after S), or S itself */
            const JDBoxPlan &p = b->bx_plans[i];
            JDBoxDesc &x = b->bx_desc[i];
            x.s_off = r.src_off; x.s_w = sw;
            for (int k = 0; k < 4; k++) x.box[k] = p.box[k];
            x.rx0 = (uint32_t)p.rx0; x.ry0 = (uint32_t)p.ry0; x.rbw = (uint32_t)(p.rx1 - p.rx0); x.rbh = (uint32_t)(p.ry1 - p.ry0);
            x.fx = (uint32_t)p.fx; x.fy = (uint32_t)p.fy;
            r.src_w = (uint32_t)p.rw; r.src_h = (uint32_t)p.rh;
            r.in_w = r.src_w; r.in_h = r.src_h;
            if (p.fx > 1 || p.fy > 1) {
                r.src_off = so;
                so += align256((size_t)r.src_w * r.src_h * bp);
                bx_ctas[1] += ((uint64_t)r.src_w * r.src_h + JD_RS_THREADS - 1) / JD_RS_THREADS;
            }
            bx_ctas[0] += ((rp.need_h ? r.dst_w : 0u) + (rp.need_v ? r.dst_h : 0u) + JD_RS_THREADS - 1) / JD_RS_THREADS;
        }
        r.mid_off = so;
        so += align256((size_t)rp.mid_bytes);
        r.coef_h = co;
        co += rp.need_h ? (uint64_t)r.dst_w * (r.ksize_h + 2) : 0;
        r.coef_v = co;
        co += rp.need_v ? (uint64_t)r.dst_h * (r.ksize_v + 2) : 0;
        const uint64_t q = ((rp.vfirst ? r.src_w : r.dst_w) + 16 / bp - 1) / (16 / bp);
        if (!b->box) ctas[0] += ((rp.need_h ? r.dst_w : 0u) + (rp.need_v ? r.dst_h : 0u) + JD_RS_THREADS - 1) / JD_RS_THREADS;
        if (rp.need_h && !rp.vfirst)   /* jdk_resize_h<4, 0>: one thread per pixel; <1, 0>: column chunks x row blocks */
            ctas[1] += bp == 4 ? ((uint64_t)r.rows * r.dst_w + JD_RS_THREADS - 1) / JD_RS_THREADS
                               : (uint64_t)((r.dst_w + JD_RS_HCOLS - 1) / JD_RS_HCOLS) * ((r.rows + JD_RS_HROWS - 1) / JD_RS_HROWS);
        ctas[2] += (q * r.dst_h + JD_RS_THREADS - 1) / JD_RS_THREADS;
        ctas[3] += rp.vfirst ? ((uint64_t)r.dst_h * r.dst_w + JD_RS_THREADS - 1) / JD_RS_THREADS : 0;
        D.descs_stage[i].out_off = b->box ? b->bx_desc[i].s_off : r.src_off;
        D.descs_stage[i].out_pitch = sw * (uint32_t)bp;
        D.descs_stage[i].out_w = sw; D.descs_stage[i].out_h = sh;
    }
    if (ctas[1] >= (1ull << 31) || ctas[2] >= (1ull << 31) || ctas[3] >= (1ull << 31) || bx_ctas[1] >= (1ull << 31)) {
        snprintf(g_err, sizeof(g_err), "resize: too many output pixels in one job");
        return 0;
    }
    for (int c = 0; c < 4; c++) D.rs_ctas[c] = (uint32_t)ctas[c];
    D.bx_ctas[0] = (uint32_t)bx_ctas[0]; D.bx_ctas[1] = (uint32_t)bx_ctas[1];
    CK(b->d_rs.alloc(&b->ctx->pool, so + 256));
    CK(b->d_rs_coef.alloc(&b->ctx->pool, co + 64));
    CK(b->d_rs_desc.alloc(&b->ctx->pool, n));
    CK(cudaMemcpyAsync(b->d_rs_desc.p, b->rs_desc.data(), sizeof(JDResizeDesc) * n, cudaMemcpyHostToDevice, b->ss.stream));
    if (b->box) {
        CK(b->d_bx_desc.alloc(&b->ctx->pool, n));
        CK(cudaMemcpyAsync(b->d_bx_desc.p, b->bx_desc.data(), sizeof(JDBoxDesc) * n, cudaMemcpyHostToDevice, b->ss.stream));
    }
    return 1;
}

/* dither: the IDCT stage writes an MCU-aligned 8-bit image into d_gray first.  Uploads the gray / output offsets and
 * pitches, the initial error lines and the band list (dbands); rewrites D.descs_stage for the IDCT stage. */
static int stage_dither(JPEGB200_BATCH *b, DecodeState &D)
{
    const int n = b->n;
    cudaStream_t st = b->ss.stream;
    std::vector<uint64_t> gray_off(3 * (size_t)n);
    std::vector<uint32_t> err_off(n);
    CK(b->d_gray.alloc(&b->ctx->pool, b->gray_total + 256));
    size_t go = 0, eo = 0;
    b->errinit.clear();
    for (int i = 0; i < n; i++) {
        const JDInfo &inf = b->infos[b->vfile[i]];
        gray_off[i] = go; err_off[i] = (uint32_t)eo;
        gray_off[(size_t)n + i] = D.descs_stage[i].out_off;         /* where jdk_dither writes the packed rows ... */
        gray_off[2 * (size_t)n + i] = D.descs_stage[i].out_pitch;   /* ... and their pitch: the caller's, or tight in the arena */
        if (b->parse_status[i] != JPEG_SUCCESS) continue;
        const uint32_t pw = (uint32_t)inf.mcus_x * (uint32_t)(inf.mcu_w >> b->sshift);
        const uint32_t ph = (uint32_t)inf.mcus_y * (uint32_t)(inf.mcu_h >> b->sshift);
        D.descs_stage[i].out_off = go;
        D.descs_stage[i].out_pitch = pw;
        go += align256((size_t)pw * ph);
        /* initial error line = the reference's DHT scratch bytes (they share usPixels, jpeg.inl:843 / :4881) */
        const size_t el = ((size_t)pw + 16 + 15) & ~(size_t)15;
        b->errinit.resize(eo + el, (uint16_t)0xFF00u);
        /* device line S[x] = errors[x + 2] */
        const size_t cp = (el + 2 < JD_HUFFVALS_BYTES) ? el : JD_HUFFVALS_BYTES - 2;
        for (size_t q = 0; q < cp; q++) b->errinit[eo + q] = (uint16_t)(0xFF00u | inf.p.huffvals[q + 2]);
        eo += el;
    }
    CK(b->d_errline.alloc(&b->ctx->pool, eo + 16));
    CK(cudaMemcpyAsync(b->d_errline.p, b->errinit.data(), eo * sizeof(uint16_t), cudaMemcpyHostToDevice, st));
    CK(b->d_gray_off.alloc(&b->ctx->pool, 3 * (size_t)n)); CK(b->d_err_off.alloc(&b->ctx->pool, n));
    /* pageable sources: the runtime stages them before returning, so the vectors may go out of scope */
    CK(cudaMemcpyAsync(b->d_gray_off.p, gray_off.data(), (size_t)n * 24, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b->d_err_off.p, err_off.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    /* one warp per band of 32 rows, band-major (band k of every image, then band k + 1): a band's producer is always
     * launched before it, and the warps resident at any time are bands that can actually run (a band may start ~113
     * steps after the one above it, so only ~W/113 bands of an image are ever active together) */
    b->dbands.clear();
    {
        /* .w: the list position of band k - 255 of the same image, which band k >= 256 waits for (jdk_dither), else ~0 */
        uint32_t maxb = 0;
        std::vector<uint32_t> nb(n, 0), prevpos(n, 0), first(n, 0);
        for (int i = 0; i < n; i++) if (b->parse_status[i] == JPEG_SUCCESS) { nb[i] = (b->descs[i].out_h + 31) / 32; if (nb[i] > maxb) maxb = nb[i]; }
        std::vector<uint32_t> where;                       /* list position of band k of image i at first[i] + k */
        for (int i = 0; i < n; i++) { first[i] = (uint32_t)where.size(); where.resize(where.size() + nb[i]); }
        for (uint32_t k = 0; k < maxb; k++)
            for (int i = 0; i < n; i++) {
                if (k >= nb[i]) continue;
                const uint32_t pos = (uint32_t)b->dbands.size();
                where[first[i] + k] = pos;
                b->dbands.push_back(make_uint4((uint32_t)i, k, prevpos[i], k >= 256 ? where[first[i] + k - 255] : ~0u));
                prevpos[i] = pos;
            }
    }
    CK(b->d_dbands.alloc(&b->ctx->pool, b->dbands.size() ? b->dbands.size() : 1)); CK(b->d_dprog.alloc(&b->ctx->pool, b->dbands.size() + 1));
    if (!b->dbands.empty()) CK(cudaMemcpyAsync(b->d_dbands.p, b->dbands.data(), b->dbands.size() * sizeof(uint4), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(b->d_dprog.p, 0, (b->dbands.size() + 1) * 4, st));
    return 1;
}

/* the entropy walk of the work list: every restart interval of the files that have restart markers */
static int run_entropy(JPEGB200_BATCH *b, DecodeState &D)
{
    if (b->work.empty()) return 1;
    cudaStream_t st = b->ss.stream;
    JDImageDesc *const fdev = b->d_fdescs.p;
    JDEntropyArgs ea;
    ea.data = b->d_comp.p; ea.imgs = fdev; ea.luts = b->d_luts.p; ea.work = b->d_work.p; ea.cta_lut = b->d_cta_lut.p;
    ea.seg_img = b->d_seg_img.p; ea.seg_start = b->d_seg_start.p; ea.blk_hdr = b->d_blk_hdr.p; ea.rec = b->d_rec.p;
    ea.seg_jmap = b->d_seg_jmap.p; ea.seg_status = b->d_seg_status.p; ea.seg_nrec = b->d_seg_nrec.p;
    ea.events = b->d_events.p; ea.event_count = b->d_counters.p; ea.event_cap = JD_EVENT_CAP;
    ea.nwork = (uint32_t)b->work.size(); ea.dc_output = (b->sshift == 3) ? 1u : (b->sshift == 2) ? 2u : 0u;
    /* default ("raw"): the entropy kernel un-stuffs in its bit reader, 64-thread CTAs.  JPEGDEC_B200_ENTROPY=clean:
     * jdk_unstuff_segs first, so that the reader is a plain word stream (128-thread CTAs).  On the H100 the raw walk is
     * the faster one (DESIGN.md 4.1). */
    static int use_clean = -1;
    if (use_clean < 0) { const char *e = getenv("JPEGDEC_B200_ENTROPY"); use_clean = (e && strcmp(e, "clean") == 0) ? 1 : 0; }
    const unsigned egrid = (unsigned)(b->work.size() / JD_ENTROPY_THREADS);
#ifdef JD_ENTROPY_PROBE
    /* development build: time the un-stuffing (clean pipeline) and the walk apart; the walk's warps print their own lines */
    cudaEvent_t pev[3];
    for (auto &e : pev) CK(cudaEventCreate(&e));
    CK(cudaEventRecord(pev[0], st));
#endif
    if (use_clean) {
        CK(b->d_clean.alloc(&b->ctx->pool, b->comp_total + 32 * (size_t)b->nseg + 4096));
        CK(b->d_seg_clen.alloc(&b->ctx->pool, b->nseg ? b->nseg : 1));
        jdk_unstuff_segs<<<(b->nseg * 32u + JD_UNSTUFF_WARPS * 32u - 1u) / (JD_UNSTUFF_WARPS * 32u), JD_UNSTUFF_WARPS * 32, 0, st>>>(
            b->d_comp.p, fdev, b->d_seg_img.p, b->d_seg_start.p, b->nseg, b->d_clean.p, b->d_seg_clen.p);
        ea.clean = b->d_clean.p; ea.seg_clen = b->d_seg_clen.p;
    } else {
        ea.clean = nullptr; ea.seg_clen = nullptr;
    }
#ifdef JD_ENTROPY_PROBE
    CK(cudaEventRecord(pev[1], st));
#endif
    const unsigned ecta = use_clean ? jd_entropy_cta_threads(true) : jd_entropy_cta_threads(false);
    const unsigned egrid_walk = egrid * (JD_ENTROPY_THREADS / ecta);
    if (use_clean) jdk_entropy<true><<<egrid_walk, ecta, 0, st>>>(ea);
    else jdk_entropy<false><<<egrid_walk, ecta, 0, st>>>(ea);
    D.launches += use_clean ? 2 : 1;
#ifdef JD_ENTROPY_PROBE
    CK(cudaEventRecord(pev[2], st));
    CK(cudaStreamSynchronize(st));
    float ms_u = 0.f, ms_w = 0.f;
    CK(cudaEventElapsedTime(&ms_u, pev[0], pev[1]));
    CK(cudaEventElapsedTime(&ms_w, pev[1], pev[2]));
    printf("JDP_LAUNCH nwork %u ctas %u unstuff_ms %.4f walk_ms %.4f\n", (unsigned)b->work.size(), egrid_walk, ms_u, ms_w);
    fflush(stdout);
    for (auto &e : pev) CK(cudaEventDestroy(e));
#endif
    return 1;
}

/* restart-free scans: un-stuff, iterate the chunk entry states to their fix point, then emit */
static int run_chunks(JPEGB200_BATCH *b, DecodeState &D)
{
    if (!b->nchunks) return 1;
    cudaStream_t st = b->ss.stream;
    JDChunkArgs ca;
    ca.comp = b->d_comp.p; ca.filt = b->d_filt.p; ca.imgs = b->d_fdescs.p; ca.luts = b->d_luts.p;
    ca.cimg_list = b->d_cimg_list.p; ca.ncimg = (uint32_t)b->cimg_list.size(); ca.flen = b->d_flen.p;
    ca.nchunks = b->nchunks;
    ca.cn = b->d_cn.p; ca.cpre = b->d_cpre.p; ca.cjmap = b->d_cjmap.p; ca.cstatus = b->d_cstatus.p; ca.cnown = b->d_cnown.p;
    ca.cdcs = b->d_cdcs.p; ca.cpe = b->d_cpe.p; ca.changed = b->d_counters.p + 2;
    ca.blk_hdr = b->d_blk_hdr.p; ca.rec = b->d_rec.p;
    ca.events = b->d_events.p; ca.event_count = b->d_counters.p; ca.event_cap = JD_EVENT_CAP;
    ca.seg_phase = b->d_seg_phase.p; ca.seg_jmap = b->d_seg_jmap.p; ca.seg_status = b->d_seg_status.p; ca.nseg_total = b->nseg;
    const unsigned gi = ((unsigned)b->cimg_list.size() * 32 + 127) / 128;
    ca.max_nch = b->max_nch; ca.Ep = b->d_Ep.p; ca.cfirst = b->d_cfirst.p;
    /* jdk_unstuff, jdk_chunk_parse and jdk_chunk_emit take their position in cimg_list from blockIdx.y, which a grid caps
     * at 65 535: a longer list runs in slices of at most that many positions, each with the list offset to its first one.
     * Every slice of a launch is on the stream before the next launch, so a parse pass still ends before the next begins. */
    const uint32_t ncimg = (uint32_t)b->cimg_list.size();
    auto sliced = [&](void (*kernel)(const JDChunkArgs), unsigned gx) {
        for (uint32_t c0 = 0; c0 < ncimg; c0 += 65535u) {
            JDChunkArgs s = ca;
            s.cimg_list = ca.cimg_list + c0;
            kernel<<<dim3(gx, std::min(ncimg - c0, 65535u)), 128, 0, st>>>(s);
            D.launches++;
        }
    };
    const unsigned gchunks = (b->max_nch + 127) / 128;
    /* guess: every chunk starts a block at its first bit (exit state of every left neighbour = (0, 0, 0)); no chunk parsed yet */
    CK(cudaMemsetAsync(b->d_E0.p, 0, (size_t)(b->nchunks + 1) * 4, st));
    CK(cudaMemsetAsync(b->d_Ep.p, 0xFE, (size_t)b->nchunks * 4, st));
    {
        const unsigned gu = ((b->max_nch * JD_CHUNK_BYTES + JD_UNSTUFF_PIECE - 1) / JD_UNSTUFF_PIECE + 3) / 4;
        sliced(jdk_unstuff<false>, gu);
        sliced(jdk_unstuff<true>, gu);
    }
    uint32_t *Xin = b->d_E0.p, *Xout = b->d_E1.p;
    int passes = 0;
    /* The entry states reach their fix point in 2-4 passes on real streams (a chunk re-synchronises well inside its 512
     * bytes), and from the third pass on only the chunks whose entry state moved are parsed again.  Normal mode:
     * JD_CHUNK_PASSES passes back to back, the last one verifying (it raises a flag if an exit state still moved) -- no
     * host round trip, so jobs of JPEGB200_decodeBatch stay in flight; batchWait re-runs the job in the iterating mode
     * below if the flag came back set. */
    static int fixed_passes = -1;   /* JPEGDEC_B200_CHUNK_PASSES=n: test hook (n = 1 forces the fallback) */
    if (fixed_passes < 0) { const char *e = getenv("JPEGDEC_B200_CHUNK_PASSES"); fixed_passes = (e && atoi(e) > 0) ? atoi(e) : JD_CHUNK_PASSES; }
    const int fixed = b->chunk_iterate ? 0 : fixed_passes;
    for (;;) {
        const int burst = fixed ? fixed : 3;
        for (int k = 0; k < burst; k++) {
            if (k == burst - 1) CK(cudaMemsetAsync(b->d_counters.p + 2, 0, 4, st));
            ca.X_in = Xin; ca.X_out = Xout;
            sliced(jdk_chunk_parse, gchunks);
            passes++;
            uint32_t *tmp = Xin; Xin = Xout; Xout = tmp;
        }
        if (fixed) break;
        CK(cudaMemcpyAsync(&b->h_changed, b->d_counters.p + 2, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (!b->h_changed || passes > (int)b->nchunks + 8) break;
    }
    ca.X_in = Xin; ca.X_out = Xout;
    jdk_chunk_prefix<<<gi, 128, 0, st>>>(ca);
    sliced(jdk_chunk_emit, gchunks);
    jdk_chunk_stitch<<<gi, 128, 0, st>>>(ca);
    D.launches += 2;
    return 1;
}

/* progressive files: one launch per wave of scan walkers */
static void run_prog_waves(JPEGB200_BATCH *b, DecodeState &D)
{
    for (size_t w = 0; w + 1 < b->pwave_off.size(); w++) {
        const uint32_t o = b->pwave_off[w], cnt = b->pwave_off[w + 1] - o;
        if (cnt == 0) continue;
        jdk_prog_scan<<<(cnt + 63) / 64, 64, 0, b->ss.stream>>>(b->d_pscans.p + o, cnt, b->d_comp.p, b->d_ptabs.p, b->d_pplanes.p, b->d_perr.p);
        D.launches++;
    }
}

/* per file: the first error of its segments (stitch), the window-truncation events (patch), and the records of the
 * progressive files from their coefficient planes (pack) */
static void run_stitch_patch_pack(JPEGB200_BATCH *b, DecodeState &D)
{
    cudaStream_t st = b->ss.stream;
    JDImageDesc *const fdev = b->d_fdescs.p;
    const int nf = b->nf;
    jdk_stitch<<<(nf + 127) / 128, 128, 0, st>>>(fdev, (uint32_t)nf, b->d_seg_jmap.p, b->d_seg_status.p, b->d_seg_phase.p, b->d_seg_nrec.p,
                                               reinterpret_cast<unsigned long long *>(b->d_counters.p + 4));
    D.launches++;
    if (!b->lj) {   /* a libjpeg decode reads the exact coefficients: no window truncation to apply */
        jdk_patch<<<32, 256, 0, st>>>(fdev, b->d_events.p, b->d_counters.p, JD_EVENT_CAP, b->d_seg_phase.p, b->d_blk_hdr.p, b->d_rec.p, b->d_counters.p + 1);
        D.launches++;
    }
    if (!b->pfiles.empty()) {
        /* after jdk_stitch, which gives a file without restart segments status 0: the pack writes the real one */
        JDProgPackArgs pa;
        pa.imgs = fdev; pa.files = b->d_pfiles.p; pa.planes = b->d_pplanes.p; pa.err_row = b->d_perr.p;
        pa.blk_hdr = b->d_blk_hdr.p; pa.rec = b->d_rec.p;
        pa.limit = b->sshift == 3 ? 1u : b->sshift == 2 ? 5u : 64u;
        pa.rec_count = reinterpret_cast<unsigned long long *>(b->d_counters.p + 4);
        jdk_prog_pack<<<(unsigned)b->pfiles.size(), 256, 0, st>>>(pa);
        D.launches++;
    }
}

/* draft views (JPEGB200_batchCreateDraft): one IDCT and one colour launch per scale present; ljd holds the scaled set of
 * descriptors (full-scale views have nmx = 0) */
static int run_lj_scaled(JPEGB200_BATCH *b, DecodeState &D, const JDLjDesc *ljd)
{
    const int n = b->n;
    cudaStream_t st = b->ss.stream;
    for (uint32_t sh = 1; sh <= 3; sh++) {
        const unsigned gb = (b->lj_s_blocks[sh] + JD_LJ_THREADS - 1) / JD_LJ_THREADS, gp = (b->lj_s_pixels[sh] + JD_LJ_THREADS - 1) / JD_LJ_THREADS;
        for (int i0 = 0; i0 < n && gb && gp; i0 += 65535) {
            const unsigned ni = (unsigned)std::min(n - i0, 65535);
            if (sh == 1) jdk_lj_idct_s<1><<<dim3(gb, ni), JD_LJ_THREADS, 0, st>>>(b->d_descs.p, ljd, b->d_blk_hdr.p, b->d_rec.p, b->d_quant.p, b->d_lj.p, (uint32_t)i0);
            else if (sh == 2) jdk_lj_idct_s<2><<<dim3(gb, ni), JD_LJ_THREADS, 0, st>>>(b->d_descs.p, ljd, b->d_blk_hdr.p, b->d_rec.p, b->d_quant.p, b->d_lj.p, (uint32_t)i0);
            else jdk_lj_idct_s<3><<<dim3(gb, ni), JD_LJ_THREADS, 0, st>>>(b->d_descs.p, ljd, b->d_blk_hdr.p, b->d_rec.p, b->d_quant.p, b->d_lj.p, (uint32_t)i0);
            if (b->ptclass == JD_PT_GRAY) jdk_lj_color_s<JD_PT_GRAY><<<dim3(gp, ni), JD_LJ_THREADS, 0, st>>>(b->d_descs.p, ljd, b->d_lj.p, D.stage_out, (uint32_t)i0, sh);
            else jdk_lj_color_s<JD_PT_8888><<<dim3(gp, ni), JD_LJ_THREADS, 0, st>>>(b->d_descs.p, ljd, b->d_lj.p, D.stage_out, (uint32_t)i0, sh);
            D.launches += 2;
        }
    }
    return 1;
}

/* libjpeg decode: planes of every image's MCU box, then upsampling + colour into the stores; images that failed keep nmx = 0 */
static int run_lj(JPEGB200_BATCH *b, DecodeState &D)
{
    const int n = b->n;
    cudaStream_t st = b->ss.stream;
    std::vector<JDLjDesc> ld = b->lj_desc;
    uint64_t po = 0;
    for (int i = 0; i < n; i++) {
        if (b->parse_status[i] != JPEG_SUCCESS) { ld[i].nmx = ld[i].nmy = 0; continue; }
        ld[i].plane_off = po;
        po += (uint64_t)b->lj_plane[i];
    }
    /* descriptors [0, n) for the full-scale kernels, [n, 2n) for the scaled ones: each set leaves the other's views empty */
    bool scaled = false;
    for (int i = 0; i < n; i++) scaled = scaled || ld[i].shift != 0;
    const int nd = scaled ? 2 * n : n;
    if (scaled) {
        ld.resize((size_t)nd);
        for (int i = 0; i < n; i++) {
            ld[n + i] = ld[i];
            if (ld[i].shift != 0) ld[i].nmx = ld[i].nmy = 0; else ld[n + i].nmx = ld[n + i].nmy = 0;
        }
    }
    CK(b->d_lj.alloc(&b->ctx->pool, po + 256));
    CK(b->d_lj_desc.alloc(&b->ctx->pool, nd));
    CK(cudaMemcpyAsync(b->d_lj_desc.p, ld.data(), sizeof(JDLjDesc) * nd, cudaMemcpyHostToDevice, st));
    if (scaled && !run_lj_scaled(b, D, b->d_lj_desc.p + n)) return 0;
    const unsigned gb = (b->lj_max_blocks + JD_LJ_THREADS - 1) / JD_LJ_THREADS, gp = (b->lj_max_pixels + JD_LJ_THREADS - 1) / JD_LJ_THREADS;
    for (int i0 = 0; i0 < n && gb && gp; i0 += 65535) {
        const unsigned ni = (unsigned)std::min(n - i0, 65535);
        jdk_lj_idct<<<dim3(gb, ni), JD_LJ_THREADS, 0, st>>>(b->d_descs.p, b->d_lj_desc.p, b->d_blk_hdr.p, b->d_rec.p, b->d_quant.p,
                                                             b->d_lj.p, (uint32_t)i0);
        if (b->ptclass == JD_PT_GRAY) jdk_lj_color<JD_PT_GRAY><<<dim3(gp, ni), JD_LJ_THREADS, 0, st>>>(b->d_descs.p, b->d_lj_desc.p, b->d_lj.p, D.stage_out, (uint32_t)i0);
        else jdk_lj_color<JD_PT_8888><<<dim3(gp, ni), JD_LJ_THREADS, 0, st>>>(b->d_descs.p, b->d_lj_desc.p, b->d_lj.p, D.stage_out, (uint32_t)i0);
        D.launches += 2;
    }
    return 1;
}

/* the IDCT + colour (or scaled) launch of images i0 .. i0 + nimg - 1, which share a geometry class, for one orientation
 * class; the grid covers max_mx x max_my MCUs per image */
static int launch_idct_run(JPEGB200_BATCH *b, const DecodeState &D, int i0, uint32_t nimg, uint32_t max_mx, uint32_t max_my, uint32_t orc)
{
    cudaStream_t st = b->ss.stream;
    const JDInfo &f = b->infos[b->vfile[i0]];
    if (b->sshift >= 2) {
        JDScaledArgs sa;
        sa.imgs = b->d_descs.p; sa.blk_hdr = b->d_blk_hdr.p; sa.rec = b->d_rec.p; sa.quant = b->d_quant.p;
        sa.out = D.stage_out; sa.img0 = (uint32_t)i0; sa.pixel_type = (uint32_t)b->pixel_type; sa.eighth = (b->sshift == 3);
        sa.padded = (b->dither_bits || b->padded) ? 1u : 0u;
        dim3 grid((max_mx * max_my + 127) / 128, nimg);
        if (orc == JD_ORC_FLIP) jdk_scaled<true, JD_ORC_FLIP><<<grid, 128, 0, st>>>(sa);
        else if (orc == JD_ORC_TRANSPOSE) jdk_scaled<true, JD_ORC_TRANSPOSE><<<grid, 128, 0, st>>>(sa);
        else if (b->roi) jdk_scaled<true><<<grid, 128, 0, st>>>(sa);
        else jdk_scaled<false><<<grid, 128, 0, st>>>(sa);
        return 1;
    }
    JDIdctArgs ia;
    ia.imgs = b->d_descs.p; ia.blk_hdr = b->d_blk_hdr.p; ia.rec = b->d_rec.p; ia.quant = b->d_quant.p;
    ia.out = D.stage_out; ia.img0 = (uint32_t)i0;
    ia.big_endian = (f.ncomp == 1) ? (b->pixel_type != RGB565_LITTLE_ENDIAN) : (b->pixel_type == RGB565_BIG_ENDIAN);
    ia.padded = (b->dither_bits || b->padded) ? 1u : 0u;
    ia.mcus_x = (uint32_t)f.mcus_x; ia.mcus_y = (uint32_t)f.mcus_y; ia.width = (uint32_t)f.width; ia.height = (uint32_t)f.height;
    ia.bpm = (uint32_t)f.bpm;
    ia.roi = b->roi ? 1u + orc : 0u;
    if (!launch_idct(ia, f.subsample, f.ncomp, b->ptclass, b->ctx->arith, b->sshift == 1, max_mx, max_my, nimg, st)) {
        snprintf(g_err, sizeof(g_err), "no kernel for subsample 0x%02x / pixel type %d", f.subsample, b->pixel_type);
        return 0;
    }
    return 1;
}

/* IDCT + colour: one launch per run of images with the same geometry class (and per orientation class of the run) */
static int run_idct(JPEGB200_BATCH *b, DecodeState &D)
{
    const int n = b->n;
    for (int i0 = 0; i0 < n;) {
        if (b->parse_status[i0] != JPEG_SUCCESS) { i0++; continue; }
        const JDInfo &f = b->infos[b->vfile[i0]];
        int i1 = i0 + 1;
        uint32_t max_mx = f.mcus_x, max_my = f.mcus_y;
        while (i1 < n && i1 - i0 < 65535 && b->parse_status[i1] == JPEG_SUCCESS) {
            const JDInfo &g = b->infos[b->vfile[i1]];
            if (g.subsample != f.subsample || g.ncomp != f.ncomp || (b->sshift < 2 && (g.width != f.width || g.height != f.height))) break;
            if ((uint32_t)g.mcus_x > max_mx) max_mx = g.mcus_x;
            if ((uint32_t)g.mcus_y > max_my) max_my = g.mcus_y;
            i1++;
        }
        if (b->roi) {
            /* the grid covers the largest box of MCUs a rectangle of the group touches, from each image's first MCU column / row */
            max_mx = max_my = 0;
            for (int i = i0; i < i1; i++) {
                const JDRoiPlan &pl = b->plans[i];
                if ((uint32_t)(pl.mcu_x1 - pl.mcu_x0 + 1) > max_mx) max_mx = (uint32_t)(pl.mcu_x1 - pl.mcu_x0 + 1);
                if ((uint32_t)(pl.mcu_y1 - pl.mcu_y0 + 1) > max_my) max_my = (uint32_t)(pl.mcu_y1 - pl.mcu_y0 + 1);
            }
        }
        /* Orientations: one instantiation per transform class.  Runs are not split by class (a loader's mix of k would cut
         * them into many small launches): each class's launch covers the whole run and its CTAs of the other class's
         * images exit at once.  The mirror kernel also stores k = 1 (no mirror); a run of k = 1 only takes the ROI kernel. */
        bool any_id = false, any_mir = false, any_tr = false;
        for (int i = i0; i < i1 && b->roi; i++) {
            const uint32_t k = b->descs[i].orient;
            if (k >= 5u) any_tr = true; else if (k >= 2u) any_mir = true; else any_id = true;
        }
        uint32_t classes[2] = {JD_ORC_NONE, JD_ORC_NONE};
        int nclass = 0;
        if (any_mir || (any_tr && any_id)) classes[nclass++] = JD_ORC_FLIP;
        else if (!any_tr) classes[nclass++] = JD_ORC_NONE;
        if (any_tr) classes[nclass++] = JD_ORC_TRANSPOSE;
        for (int ci = 0; ci < nclass; ci++) {
            /* A failed launch only leaves its error pending, and cudaFuncSetAttribute (the IDCT launchers' first-use carveout
             * calls) returns cudaSuccess and clears it (measured on an H100, CUDA runtime 12.9).  So every launch enqueued so far --
             * entropy, chunks, stitch, earlier runs -- is checked here, before the next launcher can clear its error. */
            CK(cudaGetLastError());
            if (!launch_idct_run(b, D, i0, (uint32_t)(i1 - i0), max_mx, max_my, classes[ci])) return 0;
            D.launches++;
        }
        i0 = i1;
    }
    return 1;
}

static void run_dither(JPEGB200_BATCH *b, DecodeState &D)
{
    if (b->dbands.empty()) return;
    cudaStream_t st = b->ss.stream;
    const unsigned dgrid = ((unsigned)b->dbands.size() * 32 + 127) / 128;
#define JD_DITHER_ARGS b->d_descs.p, (uint32_t)b->n, b->d_gray.p, b->d_gray_off.p, b->d_errline.p, b->d_err_off.p, D.out_base, (uint32_t)b->sshift, \
                       b->d_dbands.p, (uint32_t)b->dbands.size(), b->d_dprog.p
    if (b->dither_bits == 1) jdk_dither<1><<<dgrid, 128, 0, st>>>(JD_DITHER_ARGS);
    else if (b->dither_bits == 2) jdk_dither<2><<<dgrid, 128, 0, st>>>(JD_DITHER_ARGS);
    else jdk_dither<4><<<dgrid, 128, 0, st>>>(JD_DITHER_ARGS);
#undef JD_DITHER_ARGS
    D.launches++;
}

/* timed in the dither slot (the pixel pass after the IDCT): the two never occur together */
static void run_resize(JPEGB200_BATCH *b, DecodeState &D)
{
    cudaStream_t st = b->ss.stream;
    const uint32_t n = (uint32_t)b->n;
    const bool gray = b->ptclass == JD_PT_GRAY;
    const uint32_t *rs_ctas = D.rs_ctas;
    if (rs_ctas[0]) { jdk_resize_coeffs<<<rs_ctas[0], JD_RS_THREADS, 0, st>>>(b->d_rs_desc.p, n, b->d_rs_coef.p, b->rs_filter); D.launches++; }
    if (D.bx_ctas[1]) {   /* box batches: the reduce of S into the resize source, then the boxed tables */
        if (gray) jdk_reduce<1><<<D.bx_ctas[1], JD_RS_THREADS, 0, st>>>(b->d_rs_desc.p, b->d_bx_desc.p, n, b->d_rs.p);
        else jdk_reduce<4><<<D.bx_ctas[1], JD_RS_THREADS, 0, st>>>(b->d_rs_desc.p, b->d_bx_desc.p, n, b->d_rs.p);
        D.launches++;
    }
    if (D.bx_ctas[0]) {
        jdk_resize_coeffs_box<<<D.bx_ctas[0], JD_RS_THREADS, 0, st>>>(b->d_rs_desc.p, b->d_bx_desc.p, n, b->d_rs_coef.p, b->rs_filter);
        D.launches++;
    }
#define JD_RS_ARGS b->d_rs_desc.p, n, b->d_rs.p, b->d_rs_coef.p, D.pipe_out
    if (rs_ctas[1]) {
        if (gray) jdk_resize_h<1, 0><<<rs_ctas[1], JD_RS_THREADS, 0, st>>>(JD_RS_ARGS);
        else jdk_resize_h<4, 0><<<rs_ctas[1], JD_RS_THREADS, 0, st>>>(JD_RS_ARGS);
        D.launches++;
    }
    if (rs_ctas[2]) {
        if (gray) jdk_resize_v<1><<<rs_ctas[2], JD_RS_THREADS, 0, st>>>(JD_RS_ARGS);
        else jdk_resize_v<4><<<rs_ctas[2], JD_RS_THREADS, 0, st>>>(JD_RS_ARGS);
        D.launches++;
    }
    if (rs_ctas[3]) {   /* images whose vertical pass ran first (JDResizePlan.vfirst) */
        if (gray) jdk_resize_h<1, 1><<<rs_ctas[3], JD_RS_THREADS, 0, st>>>(JD_RS_ARGS);
        else jdk_resize_h<4, 1><<<rs_ctas[3], JD_RS_THREADS, 0, st>>>(JD_RS_ARGS);
        D.launches++;
    }
#undef JD_RS_ARGS
}

/* timed in the dither slot too, after the resize: per cut index of the operation lists, the blur pair for the views that
 * blur there, jdk_augment for the views that sharpen or move pixels with NEAREST there, jdk_augment_rs for those that
 * resample and jdk_warp for those that warp, then one jdk_augment_copy for all of them, jdk_jq_fwd (and on RGB output
 * jdk_jq_color) for the views that compress there, then jdk_color for the per-pixel operations up to the next cut */
static void run_color(JPEGB200_BATCH *b, DecodeState &D)
{
    cudaStream_t st = b->ss.stream;
    const uint32_t n = (uint32_t)b->n;
    const size_t m = b->bl_desc.size();
    for (uint32_t s = 0; s < (uint32_t)D.co_ctas.size(); s++) {
        const uint32_t f = D.bl_first[s], nb = D.bl_first[s + 1] - f;
        if (nb) {
            const JDBlurDesc *bd = b->d_bl_desc.p + f;
            const uint32_t *hb = b->d_bl_blk.p + f, *vb = b->d_bl_blk.p + m + f;
            if (b->ptclass == JD_PT_GRAY) {
                jdk_blur<1, false><<<D.bl_ctas[2 * s], JD_BL_THREADS, 0, st>>>(bd, hb, nb, D.pipe_out, b->d_bl.p);
                jdk_blur<1, true><<<D.bl_ctas[2 * s + 1], JD_BL_THREADS, 0, st>>>(bd, vb, nb, D.pipe_out, b->d_bl.p);
            } else {
                jdk_blur<4, false><<<D.bl_ctas[2 * s], JD_BL_THREADS, 0, st>>>(bd, hb, nb, D.pipe_out, b->d_bl.p);
                jdk_blur<4, true><<<D.bl_ctas[2 * s + 1], JD_BL_THREADS, 0, st>>>(bd, vb, nb, D.pipe_out, b->d_bl.p);
            }
            D.launches += 2;
        }
        const uint32_t fa = D.au_first[s], na = D.au_first[s + 1] - fa;
        if (na) {
            /* the NEAREST / sharpness entries first (nn of them, in nc CTAs), then the BILINEAR / BICUBIC ones (up to entry nr,
             * CTA nrc), then the warps */
            const JDAugDesc *ad = b->d_au_desc.p + fa;
            const uint32_t nn = D.au_nn[4 * s], nc = D.au_nn[4 * s + 1], nr = D.au_nn[4 * s + 2], nrc = D.au_nn[4 * s + 3];
            if (b->ptclass == JD_PT_GRAY) {
                if (nn) jdk_augment<1><<<nc, JD_AU_THREADS, 0, st>>>(ad, nn, D.pipe_out, b->d_bl.p);
                if (nn < nr) jdk_augment_rs<1><<<nrc - nc, JD_AU_THREADS, 0, st>>>(ad + nn, b->d_au_mat.p + fa + nn, nr - nn, nc, D.pipe_out, b->d_bl.p);
                if (nr < na) jdk_warp<1><<<D.au_ctas[s] - nrc, JD_AU_THREADS, 0, st>>>(ad + nr, b->d_au_warp.p + fa + nr, b->d_au_tab.p, na - nr, nrc, D.pipe_out, b->d_bl.p);
                jdk_augment_copy<1><<<D.au_ctas[s], JD_AU_THREADS, 0, st>>>(ad, na, D.pipe_out, b->d_bl.p);
            } else {
                if (nn) jdk_augment<4><<<nc, JD_AU_THREADS, 0, st>>>(ad, nn, D.pipe_out, b->d_bl.p);
                if (nn < nr) jdk_augment_rs<4><<<nrc - nc, JD_AU_THREADS, 0, st>>>(ad + nn, b->d_au_mat.p + fa + nn, nr - nn, nc, D.pipe_out, b->d_bl.p);
                if (nr < na) jdk_warp<4><<<D.au_ctas[s] - nrc, JD_AU_THREADS, 0, st>>>(ad + nr, b->d_au_warp.p + fa + nr, b->d_au_tab.p, na - nr, nrc, D.pipe_out, b->d_bl.p);
                jdk_augment_copy<4><<<D.au_ctas[s], JD_AU_THREADS, 0, st>>>(ad, na, D.pipe_out, b->d_bl.p);
            }
            D.launches += 1 + (nn ? 1 : 0) + (nn < nr ? 1 : 0) + (nr < na ? 1 : 0);
        }
        const uint32_t fj = D.jq_first[s], nj = D.jq_first[s + 1] - fj;
        if (nj) {
            const JDJqDesc *jd = b->d_jq_desc.p + fj;
            if (b->ptclass == JD_PT_GRAY) {
                jdk_jq_fwd<1><<<D.jq_ctas[2 * s], JD_JQ_THREADS, 0, st>>>(jd, nj, b->d_jq_tab.p, D.pipe_out, b->d_bl.p);
                D.launches++;
            } else {
                jdk_jq_fwd<4><<<D.jq_ctas[2 * s], JD_JQ_THREADS, 0, st>>>(jd, nj, b->d_jq_tab.p, D.pipe_out, b->d_bl.p);
                jdk_jq_color<<<D.jq_ctas[2 * s + 1], JD_CO_THREADS, 0, st>>>(jd, nj, D.pipe_out, b->d_bl.p);
                D.launches += 2;
            }
        }
        if (!D.co_ctas[s]) continue;
        const uint32_t *cblk = b->d_co_blk.p + (size_t)s * n;
        if (D.co_lut[s]) {
            if (b->ptclass == JD_PT_GRAY)
                jdk_color_lut<1><<<D.co_ctas[s], JD_CO_THREADS, 0, st>>>(b->d_co_desc.p, cblk, n, s, b->d_co_sum.p, D.co_nsum, D.pipe_out, D.co_hist, b->d_co_hslot.p);
            else
                jdk_color_lut<4><<<D.co_ctas[s], JD_CO_THREADS, 0, st>>>(b->d_co_desc.p, cblk, n, s, b->d_co_sum.p, D.co_nsum, D.pipe_out, D.co_hist, b->d_co_hslot.p);
        } else if (b->ptclass == JD_PT_GRAY)
            jdk_color<1><<<D.co_ctas[s], JD_CO_THREADS, 0, st>>>(b->d_co_desc.p, cblk, n, s, b->d_co_sum.p, D.co_nsum, D.pipe_out);
        else
            jdk_color<4><<<D.co_ctas[s], JD_CO_THREADS, 0, st>>>(b->d_co_desc.p, cblk, n, s, b->d_co_sum.p, D.co_nsum, D.pipe_out);
        D.launches++;
    }
}

/* timed in the dither slot too, after the resize and the colour operations */
static void run_tensor(JPEGB200_BATCH *b, DecodeState &D)
{
    if (!D.tn_ctas) return;
    cudaStream_t st = b->ss.stream;
    const uint32_t n = (uint32_t)b->n, tn_ctas = D.tn_ctas;
    const bool hwc = b->tn_spec.layout == JPEGB200_LAYOUT_HWC;
#define JD_TN_LAUNCH(ELT_, NC_)                                                                                           \
    if (hwc) jdk_tensor<ELT_, 1, NC_><<<tn_ctas, JD_TN_THREADS, 0, st>>>(b->d_tn_desc.p, n, b->d_tn.p, b->d_tn_tab.p, D.out_base); \
    else jdk_tensor<ELT_, 0, NC_><<<tn_ctas, JD_TN_THREADS, 0, st>>>(b->d_tn_desc.p, n, b->d_tn.p, b->d_tn_tab.p, D.out_base);
    if (b->tn_nc == 3) {
        if (b->tn_elt == 4) { JD_TN_LAUNCH(4, 3) } else if (b->tn_elt == 2) { JD_TN_LAUNCH(2, 3) } else { JD_TN_LAUNCH(1, 3) }
    } else {
        if (b->tn_elt == 4) { JD_TN_LAUNCH(4, 1) } else if (b->tn_elt == 2) { JD_TN_LAUNCH(2, 1) } else { JD_TN_LAUNCH(1, 1) }
    }
#undef JD_TN_LAUNCH
    D.launches++;
}

static void set_decode_counters(JPEGB200_BATCH *b, const DecodeState &D)
{
    b->counters[JPEGB200_C_LAUNCHES] = D.launches;
    b->counters[JPEGB200_C_SEGMENTS] = b->nseg_walk + b->pwalkers;
    b->counters[JPEGB200_C_BLOCKS] = (int64_t)b->nblk;
    b->counters[JPEGB200_C_COMPRESSED_BYTES] = (int64_t)b->comp_total;
    int64_t ob = 0;
    for (int i = 0; i < b->n; i++)
        if (b->parse_status[i] == JPEG_SUCCESS)
            ob += b->tensor ? JPEGB200_batchOutputBytes(b, i, nullptr) : (int64_t)b->pitches[i] * b->descs[i].out_h;
    b->counters[JPEGB200_C_OUTPUT_BYTES] = ob;
}

/* The host pipeline of one job, in stream order.  The events ev[2] .. ev[7] bound the published stage timings
 * (JPEGB200_batchWait): prescan, entropy, stitch, IDCT, and the pixel pass after it (dither, resize, colour, tensor). */
extern "C" int JPEGB200_batchDecode(JPEGB200_BATCH *b, int flags)
{
    if (!b) return 0;
    if (!b->uploaded) { snprintf(g_err, sizeof(g_err), "batchDecode before batchUpload"); return 0; }
    if (!batch_stream(b)) return 0;
    cudaStream_t st = b->ss.stream;
    const cudaEvent_t *ev = b->ss.ev;
    b->out_device = (flags & JPEGB200_OUT_DEVICE) != 0;
    b->decode_flags = flags;
    if (b->tensor && !b->out_device) {
        snprintf(g_err, sizeof(g_err), "tensor output is written to device memory only: decode with JPEGB200_OUT_DEVICE");
        return 0;
    }
    DecodeState D;
    if (!alloc_prog_planes(b) || !place_outputs(b, D)) return 0;
    /* each stage that writes through scratch redirects the stage before it: tensor <- resize <- IDCT, dither <- IDCT */
    if (b->tensor && !stage_tensor(b, D)) return 0;
    if (b->color && !stage_color(b, D)) return 0;
    if (b->resize && !stage_resize(b, D)) return 0;
    if (b->dither_bits && !stage_dither(b, D)) return 0;
    CK(cudaMemcpyAsync(b->d_descs.p, D.descs_stage.data(), sizeof(JDImageDesc) * b->n, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(b->d_counters.p, 0, 32, st));
    if (b->nchunks) CK(cudaMemsetAsync(b->d_blk_hdr.p, 0, (size_t)b->nblk * 8, st)); /* blocks a truncated restart-free scan never reaches stay empty */

    /* prescan, entropy walk, stitch and patch: one entropy-facing descriptor per file (its views share them) */
    CK(cudaEventRecord(ev[2], st));
    jdk_prescan<<<b->nf, 256, 0, st>>>(b->d_comp.p, b->d_fdescs.p, b->d_seg_start.p);
    D.launches++;
    CK(cudaEventRecord(ev[3], st));
    if (!run_entropy(b, D) || !run_chunks(b, D)) return 0;
    run_prog_waves(b, D);
    CK(cudaEventRecord(ev[4], st));
    run_stitch_patch_pack(b, D);
    CK(cudaEventRecord(ev[5], st));
    D.stage_out = b->dither_bits ? b->d_gray.p : b->resize ? b->d_rs.p : D.pipe_out;
    if (b->lj ? !run_lj(b, D) : !run_idct(b, D)) return 0;
    CK(cudaEventRecord(ev[6], st));
    if (b->dither_bits) run_dither(b, D);
    if (b->resize) run_resize(b, D);
    if (b->color) run_color(b, D);
    if (b->tensor) run_tensor(b, D);
    CK(cudaEventRecord(ev[7], st));
    CK(cudaGetLastError());
    set_decode_counters(b, D);
    return 1;
}

extern "C" int JPEGB200_batchDownload(JPEGB200_BATCH *b)
{
    if (!b || !b->ss.stream) return 0;
    cudaStream_t st = b->ss.stream;
    CK(cudaSetDevice(b->ctx->device));
    CK(cudaEventRecord(b->ss.ev[8], st));
    int64_t bytes = 0;
    if (!b->out_device) {
        const int n = b->n;
        /* one copy when the user's buffers mirror the arena layout, else one 2-D copy per image */
        bool mirror = true;
        for (int i = 0; i < n && mirror; i++) {
            if (b->parse_status[i] != JPEG_SUCCESS) continue;
            if (!b->outs[i] || !b->outs[0]) { mirror = false; break; }
            if ((uint8_t *)b->outs[i] - (uint8_t *)b->outs[0] != (ptrdiff_t)b->arena_off[i]) mirror = false;
            if (b->pitches[i] != (int64_t)b->descs[i].out_pitch) mirror = false;
        }
        int last_ok = -1;
        for (int i = n - 1; i >= 0 && last_ok < 0; i--) if (b->parse_status[i] == JPEG_SUCCESS) last_ok = i;
        if (mirror && last_ok >= 0 && b->parse_status[0] == JPEG_SUCCESS) {
            /* up to the end of the last image that has pixels (a rejected file owns no arena space) */
            size_t span = b->arena_off[last_ok] + (size_t)b->descs[last_ok].out_pitch * b->descs[last_ok].out_h;
            CK(cudaMemcpyAsync(b->outs[0], b->d_out.p, span, cudaMemcpyDeviceToHost, st));
            bytes = (int64_t)span;
        } else {
            for (int i = 0; i < n; i++) {
                if (b->parse_status[i] != JPEG_SUCCESS || !b->outs[i]) continue;
                const JDImageDesc &d = b->descs[i];
                CK(cudaMemcpy2DAsync(b->outs[i], (size_t)b->pitches[i], b->d_out.p + b->arena_off[i], d.out_pitch, d.out_pitch, d.out_h,
                                     cudaMemcpyDeviceToHost, st));
                bytes += (int64_t)d.out_pitch * d.out_h;
            }
        }
    }
    /* status and failing MCU: per file (views are judged on the host, jd_view_err_mcu) */
    if (!b->descs_dl) {
        b->descs_dl = (JDImageDesc *)b->ctx->pinpool.get(sizeof(JDImageDesc) * b->nf + 32, &b->descs_dl_bytes);
        if (!b->descs_dl) { snprintf(g_err, sizeof(g_err), "pinned status buffer allocation failed"); return 0; }
        b->h_counters = (uint32_t *)(b->descs_dl + b->nf);
    }
    CK(cudaMemcpyAsync(b->descs_dl, b->d_fdescs.p, sizeof(JDImageDesc) * b->nf, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(b->h_counters, b->d_counters.p, 32, cudaMemcpyDeviceToHost, st));
    b->downloaded = true;
    bytes += (int64_t)sizeof(JDImageDesc) * b->nf + 32;
    CK(cudaEventRecord(b->ss.ev[9], st));
    b->counters[JPEGB200_C_D2H_BYTES] = bytes;
    return 1;
}

extern "C" int JPEGB200_batchWait(JPEGB200_BATCH *b, int32_t *status)
{
    if (!b || !b->ss.stream) return 0;
    CK(cudaSetDevice(b->ctx->device));
    CK(cudaStreamSynchronize(b->ss.stream));
    CK(cudaGetLastError());
    if (b->nchunks && b->downloaded && !b->chunk_iterate && b->h_counters[2] != 0u) {
        /* a restart-free scan whose chunk entry states had not settled after the fixed passes: decode the job again,
         * iterating to the fix point */
        b->chunk_iterate = true;
        const int again = JPEGB200_batchDecode(b, b->decode_flags) && JPEGB200_batchDownload(b);
        b->chunk_iterate = false;
        if (!again) return 0;
        CK(cudaStreamSynchronize(b->ss.stream));
        CK(cudaGetLastError());
    }
    int all_ok = 1;
    /* more window-truncation events than the event buffer holds: some coefficients of this job were not patched, so its
     * pixels may differ from the reference's -- report that instead of returning them as good */
    const bool ev_overflow = b->downloaded && !b->lj && b->h_counters[0] > JD_EVENT_CAP;
    if (ev_overflow) snprintf(g_err, sizeof(g_err), "%u window-truncation events exceed the event buffer (%u): job rejected", b->h_counters[0], JD_EVENT_CAP);
    for (int i = 0; i < b->n; i++) {
        int st = b->parse_status[i];
        if (st == JPEG_SUCCESS && JPEGB200_batchErrMcu(b, i) >= 0)
            st = JPEG_DECODE_ERROR; /* jpeg.inl:5354 */
        if (st == JPEG_SUCCESS && ev_overflow) st = JPEG_DECODE_ERROR;
        if (status) status[i] = st;
        if (st != JPEG_SUCCESS) all_ok = 0;
    }
    if (b->downloaded) {
        b->counters[JPEGB200_C_EVENTS] = b->h_counters[1];            /* truncated reads the reference would have made */
        b->counters[JPEGB200_C_EVENT_CANDIDATES] = b->h_counters[0];  /* reads that are truncated for SOME start phase */
        b->counters[JPEGB200_C_RECORD_BYTES] = 2 * (int64_t)(((uint64_t)b->h_counters[5] << 32) | b->h_counters[4]);
    }
    float t;
    auto el = [&](int a, int c) { t = 0; cudaEventElapsedTime(&t, b->ss.ev[a], b->ss.ev[c]); return t; };
    b->ms[JPEGB200_T_H2D] = el(0, 1);
    b->ms[JPEGB200_T_PRESCAN] = el(2, 3);
    b->ms[JPEGB200_T_ENTROPY] = el(3, 4);
    b->ms[JPEGB200_T_STITCH] = el(4, 5);
    b->ms[JPEGB200_T_IDCT] = el(5, 6);
    b->ms[JPEGB200_T_DITHER] = el(6, 7);
    b->ms[JPEGB200_T_D2H] = el(8, 9);
    b->ms[JPEGB200_T_TOTAL] = el(2, 7);
    cudaGetLastError();
    return all_ok ? 1 : 2;
}

extern "C" int JPEGB200_batchErrMcu(JPEGB200_BATCH *b, int i)
{
    if (!b || i < 0 || i >= b->n) return -1;
    if (!b->downloaded || b->parse_status[i] != JPEG_SUCCESS) return -1;
    const JDImageDesc &fd = b->descs_dl[b->vfile[i]];
    return jd_view_err_mcu(fd.status, fd.err_mcu, b->descs[i].roi_mcu_end);
}

extern "C" int JPEGB200_batchOrientation(JPEGB200_BATCH *b, int i, int32_t *exif_tag, int32_t *applied)
{
    if (!b || i < 0 || i >= b->n) return 0;
    if (exif_tag) *exif_tag = b->exif_tag[i];
    if (applied) *applied = b->orient[i];
    return 1;
}

extern "C" int JPEGB200_batchGetTimings(JPEGB200_BATCH *b, float *ms)
{
    if (!b) return 0;
    memcpy(ms, b->ms, sizeof(b->ms));
    return 1;
}

extern "C" int JPEGB200_batchGetCounters(JPEGB200_BATCH *b, int64_t *counters)
{
    if (!b) return 0;
    memcpy(counters, b->counters, sizeof(b->counters));
    return 1;
}

/* One call for a whole batch of any size.  The batch is cut into jobs, each on its own stream, all enqueued before the
 * first wait, so that job k's pixels cross PCIe (host outputs) or its IDCT runs (device outputs) while job k+1's entropy
 * kernel runs and job k+2's compressed bytes go up.  Host outputs: jobs of JD_PIPE_IMAGES images (more when the images are
 * small), so the call costs about one D2H of the pixels instead of H2D + kernels + D2H.  Device outputs: jobs of up to
 * JD_JOB_COMP_BYTES compressed bytes, which bounds the transient coefficient records (12 B per compressed byte) however
 * large the batch is; the pixels go straight to the caller's device pointers. */
#define JD_PIPE_IMAGES 64
#define JD_PIPE_MIN_BYTES ((int64_t)64 << 20)
#define JD_PIPE_INFLIGHT 6
#define JD_JOB_COMP_BYTES ((int64_t)192 << 20)
#define JD_JOB_MAX_IMAGES 4096
#define JD_PIPE_INFLIGHT_DEVICE 3
#define JD_JOB_RESIZE_SCRATCH ((int64_t)1 << 30)
extern "C" int JPEGB200_decodeBatch(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                    int pixel_type, int options, void *const *outs, const int64_t *pitches,
                                    int flags, int32_t *status)
{
    return JPEGB200_decodeBatchROI(ctx, datas, sizes, n, pixel_type, options, nullptr, outs, pitches, flags, status);
}

extern "C" int JPEGB200_decodeBatchROI(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                       int pixel_type, int options, const int32_t *rois, void *const *outs,
                                       const int64_t *pitches, int flags, int32_t *status)
{
    return JPEGB200_decodeBatchOriented(ctx, datas, sizes, n, pixel_type, options, rois, nullptr, outs, pitches, flags, status);
}

extern "C" int JPEGB200_decodeBatchOriented(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                            int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                                            void *const *outs, const int64_t *pitches, int flags, int32_t *status)
{
    return JPEGB200_decodeBatchResized(ctx, datas, sizes, n, pixel_type, options, rois, orients, nullptr, 0, outs, pitches, flags, status);
}

extern "C" int JPEGB200_decodeBatchResized(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                           int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                                           const int32_t *out_sizes, int filter, void *const *outs, const int64_t *pitches,
                                           int flags, int32_t *status)
{
    return JPEGB200_decodeBatchTensor(ctx, datas, sizes, n, pixel_type, options, rois, orients, out_sizes, filter, nullptr, outs,
                                      pitches, nullptr, flags, status);
}

extern "C" int JPEGB200_decodeBatchTensor(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                          int pixel_type, int options, const int32_t *rois, const uint8_t *orients,
                                          const int32_t *out_sizes, int filter, const JPEGB200_TensorSpec *spec, void *const *outs,
                                          const int64_t *pitches, const int64_t *plane_strides, int flags, int32_t *status)
{
    return JPEGB200_decodeBatchViews(ctx, datas, sizes, n, nullptr, pixel_type, options, rois, orients, out_sizes, filter, spec, outs,
                                     pitches, plane_strides, flags, status);
}

extern "C" int JPEGB200_decodeBatchViews(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                         const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                         const uint8_t *orients, const int32_t *out_sizes, int filter,
                                         const JPEGB200_TensorSpec *spec, void *const *outs, const int64_t *pitches,
                                         const int64_t *plane_strides, int flags, int32_t *status)
{
    return JPEGB200_decodeBatchDraft(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, nullptr,
                                     outs, pitches, plane_strides, flags, status);
}

extern "C" int JPEGB200_decodeBatchDraft(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                         const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                         const uint8_t *orients, const int32_t *out_sizes, int filter,
                                         const JPEGB200_TensorSpec *spec, const uint8_t *draft, void *const *outs,
                                         const int64_t *pitches, const int64_t *plane_strides, int flags, int32_t *status)
{
    return JPEGB200_decodeBatchBox(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, draft,
                                   nullptr, nullptr, outs, pitches, plane_strides, flags, status);
}

extern "C" int JPEGB200_decodeBatchBox(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                       const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                       const uint8_t *orients, const int32_t *out_sizes, int filter,
                                       const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                       const double *reducing_gaps, void *const *outs, const int64_t *pitches,
                                       const int64_t *plane_strides, int flags, int32_t *status)
{
    return JPEGB200_decodeBatchColor(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, draft,
                                     boxes, reducing_gaps, nullptr, outs, pitches, plane_strides, flags, status);
}

extern "C" int JPEGB200_decodeBatchColor(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                         const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                         const uint8_t *orients, const int32_t *out_sizes, int filter,
                                         const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                         const double *reducing_gaps, const JPEGB200_ColorOp *color_ops, void *const *outs,
                                         const int64_t *pitches, const int64_t *plane_strides, int flags, int32_t *status)
{
    return JPEGB200_decodeBatchWarp(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, draft,
                                    boxes, reducing_gaps, color_ops, nullptr, outs, pitches, plane_strides, flags, status);
}

extern "C" int JPEGB200_decodeBatchWarp(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                        const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                        const uint8_t *orients, const int32_t *out_sizes, int filter,
                                        const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                        const double *reducing_gaps, const JPEGB200_ColorOp *color_ops,
                                        const JPEGB200_WarpArgs *warp_args, void *const *outs, const int64_t *pitches,
                                        const int64_t *plane_strides, int flags, int32_t *status)
{
    return JPEGB200_decodeBatchWindow(ctx, datas, sizes, n, views, pixel_type, options, rois, orients, out_sizes, filter, spec, draft,
                                      boxes, reducing_gaps, color_ops, warp_args, nullptr, outs, pitches, plane_strides, flags, status);
}

extern "C" int JPEGB200_decodeBatchWindow(JPEGB200_CTX *ctx, const uint8_t *const *datas, const int32_t *sizes, int n,
                                          const int32_t *views, int pixel_type, int options, const int32_t *rois,
                                          const uint8_t *orients, const int32_t *out_sizes, int filter,
                                          const JPEGB200_TensorSpec *spec, const uint8_t *draft, const double *boxes,
                                          const double *reducing_gaps, const JPEGB200_ColorOp *color_ops,
                                          const JPEGB200_WarpArgs *warp_args, const int32_t *windows, void *const *outs,
                                          const int64_t *pitches, const int64_t *plane_strides, int flags, int32_t *status)
{
    if (!ctx || n <= 0) return 0;
    const int64_t nv = jd_count_views(n, views, "call", g_err, (int)sizeof(g_err));   /* images (views) of the call */
    if (nv < 0) return 0;
    /* refused for the whole call, not by the first job whose views have operations */
    if (!jd_check_color(pixel_type, options, nv, color_ops, g_err, (int)sizeof(g_err))) return 0;
    const bool dev_out = (flags & JPEGB200_OUT_DEVICE) != 0;
    if (spec && !dev_out) {
        snprintf(g_err, sizeof(g_err), "tensor output is written to device memory only: call with JPEGB200_OUT_DEVICE");
        return 0;
    }
    if (dev_out && !outs) { snprintf(g_err, sizeof(g_err), "JPEGB200_decodeBatch with JPEGB200_OUT_DEVICE needs the caller's device pointers"); return 0; }
    memset(ctx->last_counters, 0, sizeof(ctx->last_counters));
    memset(ctx->last_ms, 0, sizeof(ctx->last_ms));
    ctx->last_jobs = 0;
    std::vector<JPEGB200_BATCH *> jobs;
    std::vector<int> first;
    int rc = 1, all = 1;
    size_t retired = 0;
    const size_t depth = ctx->pipe_depth ? (size_t)ctx->pipe_depth : (size_t)(dev_out ? JD_PIPE_INFLIGHT_DEVICE : JD_PIPE_INFLIGHT);
    static int64_t job_bytes = 0;   /* JPEGDEC_B200_JOB_MB=n: tuning hook for the compressed bytes per job */
    if (job_bytes == 0) { const char *e = getenv("JPEGDEC_B200_JOB_MB"); job_bytes = (e && atoi(e) > 0) ? ((int64_t)atoi(e) << 20) : JD_JOB_COMP_BYTES; }
    /* jobs complete in order; retiring one = wait + per-image status + counters + buffers back to the context's pools */
    auto retire = [&](size_t k) {
        if (rc) {
            const int r = JPEGB200_batchWait(jobs[k], status ? status + first[k] : nullptr);
            if (r == 0) all = 0; else if (r == 2 && all == 1) all = 2;
            for (int c = 0; c < JPEGB200_NUM_COUNTERS; c++) ctx->last_counters[c] += jobs[k]->counters[c];
            for (int c = 0; c < JPEGB200_NUM_TIMINGS; c++) ctx->last_ms[c] += jobs[k]->ms[c];
            ctx->last_jobs++;
        }
        JPEGB200_batchDestroy(jobs[k]);
        jobs[k] = nullptr;
    };
    static int trace = -1;          /* JPEGDEC_B200_TRACE=1: host wall clock per job on stderr (development aid) */
    if (trace < 0) { const char *e = getenv("JPEGDEC_B200_TRACE"); trace = (e && atoi(e) > 0) ? 1 : 0; }
    auto now_ms = []() { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; };
    const double t_call = trace ? now_ms() : 0.0;
    for (int i0 = 0, v0 = 0; i0 < n && rc;) {   /* i0: the job's first file, v0: its first view */
        const double t0 = trace ? now_ms() : 0.0;
        /* how many files the next job takes (cnt), with how many views (cv): jobs are cut between files only */
        int32_t cv = 0, capped = 0;
        const int maxcnt = dev_out ? JD_JOB_MAX_IMAGES : JD_PIPE_IMAGES;
        /* (measured and dropped: ramping the job size up from a small first job and down towards the end of a device-output
         * call was slower than equal jobs; every job pays the full latency of an entropy walk, so fewer, larger jobs win.) */
        const int64_t limit = job_bytes;
        const int32_t *vi = views ? views + i0 : nullptr;
        int cnt = jd_job_files(n - i0, sizes + i0, vi, maxcnt, limit, nullptr, 0, &cv, &capped);
        auto create = [&](int c) {
            return JPEGB200_batchCreateWindow(ctx, datas + i0, sizes + i0, c, vi, pixel_type, options, rois ? rois + 4 * (size_t)v0 : nullptr,
                                            orients ? orients + v0 : nullptr, out_sizes ? out_sizes + 2 * (size_t)v0 : nullptr, filter, spec,
                                            draft ? draft + v0 : nullptr, boxes ? boxes + 4 * (size_t)v0 : nullptr,
                                            reducing_gaps ? reducing_gaps + v0 : nullptr,
                                            color_ops ? color_ops + JPEGB200_COLOR_MAX_OPS * (size_t)v0 : nullptr,
                                            color_ops && warp_args ? warp_args + JPEGB200_COLOR_MAX_OPS * (size_t)v0 : nullptr,
                                            windows ? windows + 4 * (size_t)v0 : nullptr);
        };
        JPEGB200_BATCH *b = create(cnt);
        if (!b) { rc = 0; break; }
        if (!dev_out && capped) {   /* the job stopped at JD_PIPE_IMAGES views with files left */
            int64_t ob = 0;
            for (int i = 0; i < cv; i++) { int64_t pb = 0; ob += JPEGB200_batchOutputBytes(b, i, &pb); }
            if (ob < JD_PIPE_MIN_BYTES) { /* small images: redo with a job big enough to keep the kernels efficient */
                int64_t per = ob > 0 ? (ob + cv - 1) / cv : 1;
                int64_t want = (JD_PIPE_MIN_BYTES + per - 1) / per;
                int64_t cnt2 = want < nv - v0 ? want : nv - v0;
                if (cnt2 > JD_JOB_MAX_IMAGES) cnt2 = JD_JOB_MAX_IMAGES;
                int32_t cv2 = 0, capped2 = 0;
                const int c3 = jd_job_files(n - i0, sizes + i0, vi, cnt2, job_bytes, nullptr, 0, &cv2, &capped2);
                if (c3 > cnt) {
                    JPEGB200_batchDestroy(b);
                    cnt = c3; cv = cv2;
                    b = create(cnt);
                    if (!b) { rc = 0; break; }
                }
            }
        }
        if ((b->resize || b->tensor || b->pplane_total || b->lj || b->bl_scratch_total) && cnt > 1 &&
            b->rs_scratch_total + b->tn_stage_total + b->pplane_total + b->lj_plane_total + b->bl_scratch_total > JD_JOB_RESIZE_SCRATCH) {
            /* scratch of a job (resize: S + the reduced image of a box batch + intermediate; tensor: the uint8 staging; libjpeg decodes: the sample planes;
             * progressive files: the coefficient plane, counted on the file's first view; blurs: the scratch copy): at most JD_JOB_RESIZE_SCRATCH, or
             * one file with all of its views */
            std::vector<int64_t> sc(cv);
            for (int i = 0; i < cv; i++)
                sc[i] = (b->resize ? b->rs_scratch[i] : 0) + (b->tensor ? b->tn_stage[i] : 0) + (b->lj ? b->lj_plane[i] : 0) +
                        (b->color ? b->bl_scratch[i] : 0);
            for (int i = 0; i < cv; i++) if (i == 0 || b->vfile[i] != b->vfile[i - 1]) sc[i] += b->pplane[b->vfile[i]];
            int32_t cv3 = 0, capped3 = 0;
            const int c = jd_job_files(cnt, sizes + i0, vi, INT64_MAX, INT64_MAX, sc.data(), JD_JOB_RESIZE_SCRATCH, &cv3, &capped3);
            JPEGB200_batchDestroy(b);
            cnt = c; cv = cv3;
            b = create(cnt);
            if (!b) { rc = 0; break; }
        }
        jobs.push_back(b); first.push_back(v0);
        b->index_base = v0;
        const double t1 = trace ? now_ms() : 0.0;
        /* a refused pitch fails the call with batchSetOutput's message (nothing of this job is enqueued) */
        for (int i = 0; i < cv && rc; i++)
            rc = spec ? JPEGB200_batchSetOutputTensor(b, i, outs[v0 + i], pitches ? pitches[v0 + i] : 0, plane_strides ? plane_strides[v0 + i] : 0)
                      : JPEGB200_batchSetOutput(b, i, outs ? outs[v0 + i] : nullptr, pitches ? pitches[v0 + i] : 0);
        rc = rc && JPEGB200_batchUpload(b);
        const double t2 = trace ? now_ms() : 0.0;
        rc = rc && JPEGB200_batchDecode(b, flags);
        const double t3 = trace ? now_ms() : 0.0;
        rc = rc && JPEGB200_batchDownload(b);
        const double t4 = trace ? now_ms() : 0.0;
        i0 += cnt; v0 += cv;
        /* bound the device memory of a very large batch: at most `depth` jobs hold buffers at a time */
        while (rc && jobs.size() - retired > depth) retire(retired++);
        if (trace) fprintf(stderr, "[jpegdec_b200] job %zu (%d images) at %.2f ms: create %.2f upload %.2f decode %.2f download %.2f retire %.2f\n",
                           jobs.size() - 1, cv, t0 - t_call, t1 - t0, t2 - t1, t3 - t2, t4 - t3, now_ms() - t4);
    }
    { const double t5 = trace ? now_ms() : 0.0;
      while (retired < jobs.size()) retire(retired++);
      if (trace) fprintf(stderr, "[jpegdec_b200] drain %.2f ms, call %.2f ms\n", now_ms() - t5, now_ms() - t_call); }
    return rc ? all : 0;
}

extern "C" int JPEGB200_lastCallTimings(JPEGB200_CTX *ctx, float *ms, int *jobs)
{
    if (!ctx || !ms) return 0;
    memcpy(ms, ctx->last_ms, sizeof(ctx->last_ms));
    if (jobs) *jobs = ctx->last_jobs;
    return 1;
}

extern "C" int JPEGB200_lastCallCounters(JPEGB200_CTX *ctx, int64_t *counters)
{
    if (!ctx || !counters) return 0;
    memcpy(counters, ctx->last_counters, sizeof(ctx->last_counters));
    return 1;
}
