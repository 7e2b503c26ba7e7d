// sb_compositor.cpp -- fused warp + blend with every intermediate resident in HBM.
//
// One compositor is the plan of one rig: what stitcher.py:178-189 (warp_final_resolution -> Warper.warp_images,
// create_and_warp_masks, warp_rois) and stitcher.py:241-259 (Blender.prepare / feed / blend) compute for a
// fixed set of cameras.  Creation does the host geometry once (roi detection, trig tables, padded rects,
// storage); run() enqueues warp -> pyramids -> collapse for a batch of frames without touching the host.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "sb_plan.h"
#include "sb_shard.h"

namespace sb {
inline int rgbm_pitch_of(int w) { return (w + 31) & ~31; }

int make_warp_job(const Projector &p, const int rect[4], int src_w, int src_h, float *tab_dev, WarpJob *job, cudaStream_t s,
                  std::vector<float> &host_tab);
}
using namespace sb;

#define SB_PIPE_DEPTH 3  // buffer sets of the pipelined submit / wait path

// One image of the rig.  Its buffers exist when this compositor warps it (listed in sb_compositor::warped: its own block,
// on the timelapse canvas); the other images keep them null.
struct Image {
    int w = 0, h = 0;             // FINAL size: what is warped
    int in_w = 0, in_h = 0;       // the frames upload / submit take: w x h unless resized on the device
    int *taps = nullptr;          // resized on the device (sb_compositor_opts.in_w / in_h): [x taps | y taps] (resize_exact_taps)
    bool words = false;           // the warp kernel reads the source as one word per pixel, else packed u8x3 (plan_sources)
    Rect rect{};                  // fed rect (pano-absolute)
    Rect part{};                  // timelapse: the fed rect on the canvas (P_i, pano-absolute; w = h = 0 when empty)
    size_t paste_off = 0;         // timelapse: its block in Slot::paste
    WarpJob job{};                // its warp job without sources (warp_jobs adds a slot's)
    uint32_t *rgbm = nullptr;     // warped, packed; row pitch = width rounded up to 32 pixels (128-byte rows)
    float *tab = nullptr;
    float *maps = nullptr;        // projections that are not separable: xmap | ymap (built at plan time)
    uint8_t *usermask = nullptr;  // blend mask (sb_compositor_set_mask / _set_seam_mask)
    GainData gain;                // exposure gains (sb_compositor_set_gain)
};

static void image_free(Image &im, cudaStream_t s)
{
    for (void *p : {(void *)im.taps, (void *)im.rgbm, (void *)im.tab, (void *)im.maps, (void *)im.usermask}) dev_free(p, s);
    gain_free(&im.gain, s);
}

// The sources of one image in one slot (null for an image this compositor does not warp)
struct SlotImage {
    uint8_t *frame = nullptr;  // the frame as uploaded: u8x3 at the input size
    void *src = nullptr;       // what the warp reads in its place, written after every upload: the words (Image::words), or
                               // the packed FINAL-size frame of a resized image; null for a packed image that is not resized
};

// One buffer set.  Slot 0 serves upload / run / download, the timing calls and the sharded step; the pipelined
// submit / wait path deals its steps round-robin to all SB_PIPE_DEPTH slots.
struct Slot {
    std::vector<SlotImage> img;    // per image
    PanoOut out{};                 // device outputs
    // timelapse (sb_compositor_opts.timelapse): the pasted parts of the frames, one 16-byte aligned block per image with a
    // non-empty part; their k_timelapse_paste jobs; the n page-locked frames of the canvas this slot's steps end in
    uint8_t *paste = nullptr;
    PasteJob *paste_jobs = nullptr;
    uint8_t *frames = nullptr;
    cudaEvent_t e_h2d = nullptr, e_comp = nullptr, e_d2h = nullptr;  // submit: sources uploaded, step done, output downloaded
#ifndef SB_EMU
    cudaGraphExec_t graph = nullptr;  // the captured step reading this slot's buffers
#endif
};

struct sb_compositor {
    int n = 0;
    cudaStream_t stream = nullptr;
    std::vector<Image> img;            // per image
    std::vector<int> warped;           // the images this compositor warps, in launch order (set at creation)
    std::vector<ResizeJob> resize_jobs;  // scratch of prepare_sources
    std::vector<WarpJob> step_jobs;    // scratch of warp_jobs
    BlendPlan plan;
    Slot slots[SB_PIPE_DEPTH];
    int n_slots = 0;                   // slots with buffers: 1 from creation, all from the first submit on
    void *flush_buf = nullptr;
    size_t flush_bytes = 0;
    std::vector<cudaEvent_t> ev;       // ev[0] = start, ev[k+1] = after launch k
    std::vector<std::string> launch_names;
    std::vector<float> launch_ms;      // per launch, averaged over the last sb_compositor_time call
    double warp_bytes = 0;
    cudaStream_t h2d = nullptr, d2h = nullptr;  // copy streams of the pipelined path
    unsigned long long submitted = 0;
    unsigned graph_kernels = 0;
    std::vector<cudaEvent_t> tev;  // step start / end events of sb_compositor_time
    // multi-GPU: this process composites images [first, first + count) and one column strip of the panorama
    bool sharded = false;
    int first = 0, count = 0;
    ShardPlan shard;
    // timelapse mode: no blend plan; every step writes one frame of the canvas per image (cv.detail.Timelapser)
    int timelapse = 0;                 // 0, SB_TIMELAPSE_AS_IS or SB_TIMELAPSE_CROP
    Rect canvas{0, 0, 0, 0};           // resultRoi / resultRoiIntersection of the fed rects (pano-absolute)
    size_t paste_bytes = 0;
    long long paste_max = 0;           // largest 3 * |P_i|
    double paste_model = 0;            // model bytes of k_timelapse_paste
};

// the sources of the warped images and an output of slot 0's size (the panorama, or this rank's strip)
static int slot_alloc(sb_compositor *c, Slot &sl)
{
    cudaStream_t s = c->stream;
    sl.img.assign(c->n, SlotImage{});
    for (int i : c->warped) {
        const Image &im = c->img[i];
        SlotImage &si = sl.img[i];
        const size_t px = (size_t)im.w * im.h;
        SB_TRY(dev_alloc((void **)&si.frame, (size_t)im.in_w * im.in_h * 3 + SB_SRC_PAD, s));
        if (im.words)
            SB_TRY(dev_alloc(&si.src, (px + 4) * sizeof(uint32_t), s));
        else if (im.taps)
            SB_TRY(dev_alloc(&si.src, px * 3 + SB_SRC_PAD, s));
    }
    SB_CUDA(cudaEventCreateWithFlags(&sl.e_h2d, cudaEventDisableTiming));
    SB_CUDA(cudaEventCreateWithFlags(&sl.e_comp, cudaEventDisableTiming));
    SB_CUDA(cudaEventCreateWithFlags(&sl.e_d2h, cudaEventDisableTiming));
    if (c->timelapse) {
        if (c->warped.empty()) return SB_OK;
        SB_TRY(dev_alloc((void **)&sl.paste, c->paste_bytes, s));
        std::vector<PasteJob> pj;
        for (int i : c->warped) {
            const Image &im = c->img[i];
            pj.push_back(PasteJob{im.rgbm, sl.paste + im.paste_off, rgbm_pitch_of(im.part.w), im.part.w, im.part.h});
        }
        SB_TRY(dev_alloc((void **)&sl.paste_jobs, pj.size() * sizeof(PasteJob), s));
        SB_CUDA(cudaMemcpyAsync(sl.paste_jobs, pj.data(), pj.size() * sizeof(PasteJob), cudaMemcpyHostToDevice, s));
        SB_CUDA(cudaStreamSynchronize(s));  // pj goes out of scope
        return SB_OK;
    }
    PanoOut &o = sl.out;
    o.w = c->slots[0].out.w;
    o.h = c->slots[0].out.h;
    o.rgb_pitch = (long long)o.w * 3;
    o.mask_pitch = o.w;
    SB_TRY(dev_alloc((void **)&o.rgb, (size_t)std::max(o.w, 1) * 3 * std::max(o.h, 1), s));
    SB_TRY(dev_alloc((void **)&o.mask, (size_t)std::max(o.w, 1) * std::max(o.h, 1), s));
    return SB_OK;
}

static void slot_free(Slot &sl, cudaStream_t s)
{
    for (SlotImage &si : sl.img) {
        dev_free(si.frame, s);
        dev_free(si.src, s);
    }
    dev_free(sl.out.rgb, s);
    dev_free(sl.out.mask, s);
    dev_free(sl.paste, s);
    dev_free(sl.paste_jobs, s);
    if (sl.frames) (void)cudaFreeHost(sl.frames);
    for (cudaEvent_t e : {sl.e_h2d, sl.e_comp, sl.e_d2h})
        if (e) (void)cudaEventDestroy(e);
#ifndef SB_EMU
    if (sl.graph) (void)cudaGraphExecDestroy(sl.graph);
#endif
}

static void compositor_free(sb_compositor *c)
{
    if (!c) return;
    cudaStream_t s = c->stream ? c->stream : default_stream();
    for (cudaStream_t q : {c->stream, c->h2d, c->d2h})  // nothing queued may still use what is freed
        if (q) (void)cudaStreamSynchronize(q);
    for (Slot &sl : c->slots) slot_free(sl, s);
    for (Image &im : c->img) image_free(im, s);
    dev_free(c->flush_buf, s);
    if (c->h2d) (void)cudaStreamDestroy(c->h2d);
    if (c->d2h) (void)cudaStreamDestroy(c->d2h);
    for (auto &e : c->tev) (void)cudaEventDestroy(e);
    c->shard.release(s);
    c->plan.release(s);
    for (auto &e : c->ev)
        if (e) (void)cudaEventDestroy(e);
    if (c->stream) {
        (void)cudaStreamSynchronize(c->stream);
        (void)cudaStreamDestroy(c->stream);
    }
    delete c;
}

// What image i feeds with a crop (Stitcher.crop_final_resolution): the slice rect = (x, y, w, h) of its warped image,
// clipped at the bottom and right like a numpy slice, is warped -- `proj` in pano-absolute coordinates -- and fed at
// (corner, fed size); the prepared size only enters the pano roi.  The rounding of the two scaled rectangles differs, so
// neither the slice nor the corner can be derived from the other.
static int crop_image(const sb_crop *crop, int i, const Rect &warped, Rect *proj, Rect *placed, int prepared[2])
{
    const int *r = crop->rect + 4 * i;
    const int *sz = crop->size + 2 * i;
    if (r[0] < 0 || r[1] < 0 || r[2] < 0 || r[3] < 0 || sz[0] < 0 || sz[1] < 0) {
        set_error("compositor: crop of image %d has a negative offset or size (%d,%d %dx%d, size %dx%d)", i, r[0], r[1], r[2], r[3], sz[0], sz[1]);
        return SB_ERR_INVALID;
    }
    const int w = std::max(0, std::min(r[2], warped.w - r[0])), h = std::max(0, std::min(r[3], warped.h - r[1]));
    if (w == 0 || h == 0) {
        // the reference's blenders cannot take an empty image either: feed asserts (no, feather) or never returns (multiband)
        set_error("compositor: crop of image %d is empty (%d,%d %dx%d of a %dx%d warped image)", i, r[0], r[1], r[2], r[3], warped.w, warped.h);
        return SB_ERR_INVALID;
    }
    if (w > sz[0] || h > sz[1]) {
        set_error("compositor: crop of image %d feeds %dx%d, more than its prepared size %dx%d", i, w, h, sz[0], sz[1]);
        return SB_ERR_INVALID;
    }
    *proj = Rect{warped.x + r[0], warped.y + r[1], w, h};
    *placed = Rect{crop->corner[2 * i], crop->corner[2 * i + 1], w, h};
    prepared[0] = sz[0];
    prepared[1] = sz[1];
    return SB_OK;
}

// Images.resize_img_by_scaler sizes: the reference resizes camera frames to the FINAL sizes with cv.resize and never
// scales up (MegapixDownscaler); the staging buffers hold the frames, so they obey the compositor's source limit
static int check_input_sizes(const sb_rig *rig, const int *in_w, const int *in_h)
{
    for (int i = 0; i < rig->n_images; ++i) {
        const int w = in_w[i], h = in_h[i], fw = rig->src_w[i], fh = rig->src_h[i];
        if (w <= 0 || h <= 0) {
            set_error("compositor: input frame of image %d has the size %dx%d", i, w, h);
            return SB_ERR_INVALID;
        }
        if (w >= SB_MAX_WARP_SIDE || h >= SB_MAX_WARP_SIDE) {
            set_error("compositor: input frame of image %d (%dx%d) has a side of %d px or more", i, w, h, SB_MAX_WARP_SIDE);
            return SB_ERR_INVALID;
        }
        if (w < fw || h < fh) {
            set_error("compositor: input frame of image %d (%dx%d) is smaller than its FINAL size %dx%d on some axis; frames are "
                      "only scaled down", i, w, h, fw, fh);
            return SB_ERR_INVALID;
        }
    }
    return SB_OK;
}

// The source the warp kernel reads, chosen once per warped image, and the taps of the images resized on the device.
// launch_warp picks its kernel per batch of SB_WARP_BATCH jobs of `warped`, and only the RGBM kernel reads words: the
// images of such a batch read words (unless SB_SRC4=0), those of a k_warp_wide batch (a map projection or a 1-px side
// in the batch) read packed u8x3.  slot_alloc allocates only the buffer that is read.
static int plan_sources(sb_compositor *c, cudaStream_t s)
{
    const char *e = getenv("SB_SRC4");  // SB_SRC4=0: the warp kernel reads the packed 3-byte sources (A/B switch)
    const bool src4 = !(e && e[0] == '0');
    const std::vector<int> &order = c->warped;
    std::vector<WarpJob> jobs;
    for (int i : order) jobs.push_back(c->img[i].job);
    for (size_t b = 0; b < order.size(); b += SB_WARP_BATCH) {
        const int cnt = (int)std::min<size_t>(SB_WARP_BATCH, order.size() - b);
        const bool words = src4 && warp_batch_rgbm(jobs.data() + b, cnt);
        for (int k = 0; k < cnt; ++k) c->img[order[b + k]].words = words;
    }
    std::vector<int> t;
    for (int i : order) {
        Image &im = c->img[i];
        if (im.in_w == im.w && im.in_h == im.h) continue;
        t.resize((size_t)3 * (im.w + im.h));
        resize_exact_taps(im.in_w, im.w, t.data());
        resize_exact_taps(im.in_h, im.h, t.data() + (size_t)3 * im.w);
        SB_TRY(dev_alloc((void **)&im.taps, t.size() * sizeof(int), s));
        SB_CUDA(cudaMemcpyAsync(im.taps, t.data(), t.size() * sizeof(int), cudaMemcpyHostToDevice, s));
        SB_CUDA(cudaStreamSynchronize(s));  // t is reused by the next image
    }
    return SB_OK;
}

// image i has buffers here: this compositor warps it
static bool warped_here(const sb_compositor *c, int i) { return c->img[i].rgbm != nullptr; }

// After the frames of images [i0, i1) have reached `sl` (in the order of stream s): the sources the warp kernel reads in
// their place -- the repack into words, or for a resized image k_resize_src into either layout, one launch for all of them
static int prepare_sources(sb_compositor *c, const Slot &sl, int i0, int i1, cudaStream_t s)
{
    c->resize_jobs.clear();
    for (int i = i0; i < i1; ++i) {
        const Image &im = c->img[i];
        const SlotImage &si = sl.img[i];
        uint32_t *words = im.words ? (uint32_t *)si.src : nullptr;
        if (im.taps)  // {src, dst4, dst3, tx, ty, sw, dw, px}
            c->resize_jobs.push_back(ResizeJob{si.frame, words, words ? nullptr : (uint8_t *)si.src, im.taps, im.taps + (size_t)3 * im.w,
                                               im.in_w, im.w, (long long)im.w * im.h});
        else if (words)
            SB_TRY(launch_repack_rgbx(si.frame, words, (long long)im.w * im.h, s));
    }
    return c->resize_jobs.empty() ? SB_OK : launch_resize_src(c->resize_jobs.data(), (int)c->resize_jobs.size(), s);
}

// Timelapser.initialize(corners, sizes) (timelapser.py:36-37) over what Blender.prepare would have received -- the warped
// rects, or with a crop the crop corners and prepared sizes: the canvas is resultRoi ("as_is") or resultRoiIntersection
// ("crop"), which builds cv::Rect(tl, br) and so returns an empty intersection as the gap between the images.  Frame i
// shows the part P_i of fed image i that lands on the canvas; only P_i is warped (its rect in `proj` narrowed to it) and
// pasted.  An image with an empty P_i gives an all-zero frame and no work.
static int plan_timelapse(sb_compositor *c, int kind, const int *corners, const int *sizes, Rect *proj)
{
    const int n = c->n;
    Rect &cv = c->canvas;
    if (kind == SB_TIMELAPSE_AS_IS) {
        cv = result_roi(corners, sizes, n);
    } else {
        int tlx = corners[0], tly = corners[1], brx = corners[0] + sizes[0], bry = corners[1] + sizes[1];
        for (int i = 1; i < n; ++i) {
            tlx = std::max(tlx, corners[2 * i]);
            tly = std::max(tly, corners[2 * i + 1]);
            brx = std::min(brx, corners[2 * i] + sizes[2 * i]);
            bry = std::min(bry, corners[2 * i + 1] + sizes[2 * i + 1]);
        }
        cv = Rect{std::min(tlx, brx), std::min(tly, bry), std::abs(brx - tlx), std::abs(bry - tly)};
    }
    if (cv.w <= 0 || cv.h <= 0) {
        // the reference's Timelapser cannot show it either: get_frame fails in convertScaleAbs
        set_error("compositor: the timelapse canvas (%d,%d %dx%d) has a zero side", cv.x, cv.y, cv.w, cv.h);
        return SB_ERR_INVALID;
    }
    for (int i = 0; i < n; ++i) {
        Image &im = c->img[i];
        const Rect &r = im.rect;
        const int x0 = std::max(r.x, cv.x), y0 = std::max(r.y, cv.y);
        const int x1 = std::min(r.x + r.w, cv.x + cv.w), y1 = std::min(r.y + r.h, cv.y + cv.h);
        if (x1 <= x0 || y1 <= y0) continue;
        im.part = Rect{x0, y0, x1 - x0, y1 - y0};
        proj[i] = Rect{proj[i].x + x0 - r.x, proj[i].y + y0 - r.y, x1 - x0, y1 - y0};
        const long long bytes = 3ll * (x1 - x0) * (y1 - y0);
        im.paste_off = c->paste_bytes;
        c->paste_bytes += ((size_t)bytes + 15) & ~(size_t)15;
        c->paste_max = std::max(c->paste_max, bytes);
        c->paste_model += 7.0 * (x1 - x0) * (y1 - y0);  // RGBM words read, u8x3 written
    }
    return SB_OK;
}

// `o` has passed valid_opts
static int compositor_build(sb_compositor *c, const sb_rig *rig, const sb_compositor_opts &o)
{
    const int *in_w = o.in_w, *in_h = o.in_h;
    const sb_crop *crop = o.crop;
    c->timelapse = o.timelapse;
    const int n = rig->n_images;
    c->n = n;
    c->sharded = o.world > 1;
    c->first = 0;
    c->count = n;
    if (c->sharded) ShardPlan::block_of(n, o.world, o.rank, &c->first, &c->count);
    SB_TRY(ensure_device());
    SB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    cudaStream_t s = c->stream;

    if (in_w) SB_TRY(check_input_sizes(rig, in_w, in_h));
    c->img.resize(n);
    std::vector<int> corners(2 * n), sizes(2 * n);
    std::vector<Rect> proj(n);  // the pano-absolute rect image i is warped over
    std::vector<Projector> projs(n);
    for (int i = 0; i < n; ++i) {
        Image &im = c->img[i];
        im.w = rig->src_w[i];
        im.h = rig->src_h[i];
        im.in_w = in_w ? in_w[i] : im.w;
        im.in_h = in_h ? in_h[i] : im.h;
        Projector &p = projs[i];
        projector_setup(p, rig->warp_type, rig->scale, rig->K + 9 * i, rig->R + 9 * i);
        int rect[4];
        projector_roi(p, im.w, im.h, rect);
        if (rect[2] <= 0 || rect[3] <= 0 || (long long)rect[2] * rect[3] > (1ll << 31)) {
            set_error("compositor: degenerate warped roi %dx%d for image %d", rect[2], rect[3], i);
            return SB_ERR_INVALID;
        }
        // the reference warps every image whole (before any crop) with cv::remap, which refuses such sides
        if (im.w >= SB_MAX_WARP_SIDE || im.h >= SB_MAX_WARP_SIDE || rect[2] >= SB_MAX_WARP_SIDE || rect[3] >= SB_MAX_WARP_SIDE) {
            set_error("compositor: image %d (source %dx%d, warped %dx%d) has a side of %d px or more, which cv::remap refuses", i,
                      im.w, im.h, rect[2], rect[3], SB_MAX_WARP_SIDE);
            return SB_ERR_INVALID;
        }
        im.rect = Rect{rect[0], rect[1], rect[2], rect[3]};
        corners[2 * i] = rect[0];
        corners[2 * i + 1] = rect[1];
        sizes[2 * i] = rect[2];
        sizes[2 * i + 1] = rect[3];
        if (crop) {  // from here on `rect` is the part of the warped rect that is warped and fed, im.rect where it is fed
            Rect slice;
            SB_TRY(crop_image(crop, i, im.rect, &slice, &im.rect, &sizes[2 * i]));
            rect[0] = slice.x;
            rect[1] = slice.y;
            rect[2] = slice.w;
            rect[3] = slice.h;
            corners[2 * i] = im.rect.x;
            corners[2 * i + 1] = im.rect.y;
        }
        proj[i] = Rect{rect[0], rect[1], rect[2], rect[3]};
    }
    if (c->timelapse) SB_TRY(plan_timelapse(c, c->timelapse, corners.data(), sizes.data(), proj.data()));
    // the images this compositor warps: its block, less those off the timelapse canvas (neither uploaded nor warped)
    for (int i = c->first; i < c->first + c->count; ++i)
        if (!c->timelapse || c->img[i].part.w > 0) c->warped.push_back(i);
    std::vector<float> host_tab;
    for (int i : c->warped) {
        Image &im = c->img[i];
        const Projector &p = projs[i];
        int rect[4] = {proj[i].x, proj[i].y, proj[i].w, proj[i].h};
        SB_TRY(dev_alloc((void **)&im.rgbm, (size_t)rgbm_pitch_of(rect[2]) * rect[3] * 4, s));
        // the row padding (never written by the warp kernel) is read by the tile kernels' 16-byte copies: weight 0
        SB_CUDA(cudaMemsetAsync(im.rgbm, 0, (size_t)rgbm_pitch_of(rect[2]) * rect[3] * 4, s));
        SB_TRY(dev_alloc((void **)&im.tab, warp_table_floats(rect[2], rect[3]) * sizeof(float), s));
        SB_TRY(make_warp_job(p, rect, im.w, im.h, im.tab, &im.job, s, host_tab));
        SB_CUDA(cudaStreamSynchronize(s));  // host_tab is reused by the next image
        if (projector_needs_maps(p)) {
            SB_TRY(dev_alloc((void **)&im.maps, (size_t)2 * rect[2] * rect[3] * sizeof(float), s));
            SB_TRY(warp_maps_upload(p, rect, im.maps, &im.job, s));
        }
        im.job.spitch = (long long)im.w * 3;
        im.job.dst_rgbm = im.rgbm;
        im.job.rgbm_pitch = rgbm_pitch_of(rect[2]);
        c->warp_bytes += 3.0 * im.w * im.h + 4.0 * rect[2] * rect[3];
    }
    if (!c->timelapse) {  // a timelapse has no blend plan: its step is warp -> paste into the slot's frames
        // Blender.prepare (blender.py:23-38)
        const Rect roi = result_roi(corners.data(), sizes.data(), n);
        int kind, nbr;
        float sharp;
        derive_blend_params(rig->blend_kind, rig->blend_strength, roi, &kind, &nbr, &sharp);
        SB_TRY(c->plan.set_geometry(kind, nbr, sharp, roi));
        {
            // the mask byte of a warped pixel is the validity test's 0 / 255 until a caller supplies masks (SB_PD_BIN=0: A/B switch)
            const char *e = getenv("SB_PD_BIN");
            c->plan.binary_masks = !(e && e[0] == '0');
        }
        for (const Image &im : c->img) {
            FeedDesc f;
            std::memset(&f, 0, sizeof f);
            f.w = im.rect.w;
            f.h = im.rect.h;
            f.tlx = im.rect.x;
            f.tly = im.rect.y;
            f.rgbm = im.rgbm;
            f.rgbm_pitch = rgbm_pitch_of(im.rect.w);
            SB_TRY(c->plan.add_feed(f));
        }
        int out_w = roi.w, out_h = roi.h;
        if (c->sharded) {
            c->plan.active_first = c->first;
            c->plan.active_count = c->count;
            SB_TRY(c->shard.build(c->plan, o.rank, o.world));
            int lo, hi;
            c->shard.strip(c->plan, &lo, &hi);
            if (c->shard.axis == 0)
                out_w = hi - lo;
            else
                out_h = hi - lo;  // row strips (feather, image blocks stacked vertically)
        }
        SB_TRY(c->plan.allocate(s));
        if (c->sharded) SB_TRY(c->shard.allocate(c->plan, s));
        c->slots[0].out.w = out_w;
        c->slots[0].out.h = out_h;
    }
    SB_TRY(plan_sources(c, s));
    SB_TRY(slot_alloc(c, c->slots[0]));
    c->n_slots = 1;
    SB_CUDA(cudaStreamSynchronize(s));
    return SB_OK;
}

// the warp jobs of one step on `slot`: those of the warped images, in launch order, with the slot's sources (built in a
// scratch vector: no allocation per step); c->warped.size() of them
static const WarpJob *warp_jobs(sb_compositor *c, int slot)
{
    const Slot &sl = c->slots[slot];
    c->step_jobs.clear();
    for (int i : c->warped) {
        const Image &im = c->img[i];
        const SlotImage &si = sl.img[i];
        WarpJob j = im.job;
        j.src4 = im.words ? (const uint32_t *)si.src : nullptr;
        j.src = im.words ? nullptr : im.taps ? (const uint8_t *)si.src : si.frame;
        c->step_jobs.push_back(j);
    }
    return c->step_jobs.data();
}

// the jobs are baked into the captured steps: capture again on next use
static void drop_graphs(sb_compositor *c)
{
#ifndef SB_EMU
    for (Slot &sl : c->slots)
        if (sl.graph) {
            (void)cudaGraphExecDestroy(sl.graph);
            sl.graph = nullptr;
        }
#endif
}

// image i blends with the mask in its usermask: stored as its weight byte (and_validity 0) or ANDed with the
// warped validity mask (1); the mask may hold gray values
static void use_blend_mask(sb_compositor *c, int i, int and_validity)
{
    Image &im = c->img[i];
    im.job.blend_mask = im.usermask;
    im.job.blend_mask_pitch = im.rect.w;
    im.job.blend_mask_and = and_validity;
    c->plan.binary_masks = false;
    drop_graphs(c);
}

static int download_out(const PanoOut &o, uint8_t *dst, size_t dst_pitch, uint8_t *dst_mask, size_t mask_pitch, cudaStream_t s)
{
    if (dst) SB_CUDA(sb_copy2d(dst, dst_pitch, o.rgb, (size_t)o.rgb_pitch, (size_t)o.w * 3, o.h, cudaMemcpyDeviceToHost, s));
    if (dst_mask) SB_CUDA(sb_copy2d(dst_mask, mask_pitch, o.mask, (size_t)o.mask_pitch, o.w, o.h, cudaMemcpyDeviceToHost, s));
    return SB_OK;
}

static int compositor_enqueue_kernels(sb_compositor *c, bool events, int slot);

// One step = one CUDA graph launch: the plan is static, so the ~2(nb+1) kernel launches are captured once per
// buffer slot and replayed (the coarse levels are launch-latency bound).  SB_GRAPH=0 launches them one by one.
static int compositor_enqueue(sb_compositor *c, bool events, int slot = 0)
{
#ifndef SB_EMU
    static const bool use_graph = [] {
        const char *e = getenv("SB_GRAPH");
        return !(e && e[0] == '0');
    }();
    if (!events && use_graph && !c->sharded) {  // (the sharded step contains the NCCL exchange: launched directly)
        cudaStream_t s = c->stream;
        if (!c->slots[slot].graph) {
            const unsigned long long before = sb_launch_count();
            SB_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
            const int rc = compositor_enqueue_kernels(c, false, slot);
            cudaGraph_t g = nullptr;
            const cudaError_t e = cudaStreamEndCapture(s, &g);
            c->graph_kernels = (unsigned)(sb_launch_count() - before);
            adjust_launch_count(-(long long)c->graph_kernels);  // captured, not executed
            if (rc != SB_OK) {
                if (g) (void)cudaGraphDestroy(g);
                return rc;
            }
            if (e != cudaSuccess) return cuda_fail(e, "cudaStreamEndCapture", __FILE__, __LINE__);
            const cudaError_t ei = cudaGraphInstantiate(&c->slots[slot].graph, g, 0);
            (void)cudaGraphDestroy(g);
            if (ei != cudaSuccess) return cuda_fail(ei, "cudaGraphInstantiate", __FILE__, __LINE__);
        }
        SB_CUDA(cudaGraphLaunch(c->slots[slot].graph, s));
        adjust_launch_count((long long)c->graph_kernels);
        return SB_OK;
    }
#endif
    return compositor_enqueue_kernels(c, events, slot);
}

// The sharded step's two loops (sb_shard.h); `transport` false leaves out guard, send_part, receive_part and consumed (the
// transport hooks move the slabs themselves).  Loop 0, each exchange part in order: the own images' work its partial sums
// read (feather weights, or the pyrDowns to the part's levels), the partial sums, the send.
template <class Mark>
static int shard_send_parts(sb_compositor *c, bool transport, cudaStream_t s, const Mark &mark)
{
    BlendPlan &P = c->plan;
    ShardPlan &sh = c->shard;
    for (int part = 0; part < sh.parts(); ++part) {
        if (sh.feather) {
            SB_TRY(launch_feather_weights(P.imgs_dev + c->first, P.imgs.data() + c->first, c->count, P.sharpness, s));
            SB_TRY(mark("feather_weights"));
        } else {
            for (int l = part == 0 ? 0 : 1; l < (part == 0 ? 1 : P.nb); ++l) {
                SB_TRY(P.pyrdown(l, c->first, c->count, s));
                SB_TRY(mark("pyrdown_l" + std::to_string(l)));
            }
        }
        if (transport && part == 0) SB_TRY(sh.guard(s));
        SB_TRY(sh.partial_out(P, part, s));
        SB_TRY(mark(sh.feather ? "partial_out" : part == 0 ? "partial_l0" : "partial_coarse"));
        if (transport) SB_TRY(sh.send_part(part, s));
    }
    return SB_OK;
}

// loop 1, coarsest part first: the receive and the finish of the own strip into `out`
template <class Mark>
static int shard_finish_parts(sb_compositor *c, const PanoOut &out, bool transport, cudaStream_t s, const Mark &mark)
{
    ShardPlan &sh = c->shard;
    for (int part = sh.parts() - 1; part >= 0; --part) {
        if (transport) SB_TRY(sh.receive_part(part, s));
        SB_TRY(sh.finish(c->plan, out, part, s));
        if (transport && part == 0) SB_TRY(sh.consumed(s));
        SB_TRY(mark(sh.feather ? "feather_finish" : part == 0 ? "finish_l0" : "finish_coarse"));  // includes waiting for the slabs
    }
    return SB_OK;
}

static int compositor_enqueue_kernels(sb_compositor *c, bool events, int slot)
{
    cudaStream_t s = c->stream;
    size_t k = 0;
    auto mark = [&](const std::string &name) -> int {
        if (!events) return SB_OK;
        if (c->ev.size() <= k) {
            cudaEvent_t e;
            SB_CUDA(cudaEventCreate(&e));
            c->ev.push_back(e);
        }
        SB_CUDA(cudaEventRecord(c->ev[k], s));
        if (k > 0) {
            if (c->launch_names.size() < k) c->launch_names.push_back(name);
        }
        ++k;
        return SB_OK;
    };
    SB_TRY(mark("start"));
    SB_TRY(launch_warp(warp_jobs(c, slot), (int)c->warped.size(), s));
    SB_TRY(mark("warp"));
    if (c->timelapse) {
        SB_TRY(launch_timelapse_paste(c->slots[slot].paste_jobs, (int)c->warped.size(), c->paste_max, s));
        return mark("paste");
    }
    const PanoOut &out = c->slots[slot].out;
    if (!c->sharded) return c->plan.run(out, s, events ? std::function<int(const std::string &)>(mark) : nullptr);
    SB_TRY(shard_send_parts(c, true, s, mark));
    return shard_finish_parts(c, out, true, s, mark);
}

// every slot has its buffers (and a timelapse its frames): the pipelined path may run
static bool pipe_ready(const sb_compositor *c)
{
    if (c->n_slots < SB_PIPE_DEPTH) return false;
    if (c->timelapse)
        for (const Slot &sl : c->slots)
            if (!sl.frames) return false;
    return true;
}

// the other slots and the copy streams of sb_compositor_submit / _wait, on the first submit; after a failure the next
// submit picks up where this one stopped
static int compositor_pipe_init(sb_compositor *c)
{
    if (!c->h2d) SB_CUDA(cudaStreamCreateWithFlags(&c->h2d, cudaStreamNonBlocking));
    if (!c->d2h) SB_CUDA(cudaStreamCreateWithFlags(&c->d2h, cudaStreamNonBlocking));
    for (; c->n_slots < SB_PIPE_DEPTH; ++c->n_slots) SB_TRY(slot_alloc(c, c->slots[c->n_slots]));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    if (c->timelapse) {
        // the frames every timelapse step ends in: zeroed once; each step then writes only the parts P_i
        const size_t frame = (size_t)c->canvas.w * c->canvas.h * 3, bytes = frame * c->n;
        for (Slot &sl : c->slots) {
            if (sl.frames) continue;
            if (host_alloc_pinned((void **)&sl.frames, bytes) != cudaSuccess) {
                set_error("sb_compositor_submit_timelapse: %zu bytes of page-locked memory for the frames (%d slots x %d frames of "
                          "%dx%d x 3 bytes) could not be allocated", bytes * SB_PIPE_DEPTH, SB_PIPE_DEPTH, c->n, c->canvas.w, c->canvas.h);
                return SB_ERR_NOMEM;
            }
            std::memset(sl.frames, 0, bytes);
        }
    }
    return SB_OK;
}

// One pipelined step of sb_compositor_submit / _submit_timelapse (`what`) on the next slot: H2D of the warped images,
// the step, and `download`'s D2H of the slot's output are enqueued on three streams and chained with events; with three
// buffer sets the copies of a step overlap the kernels and copies of its neighbours.
static int pipe_step(sb_compositor *c, const char *what, const uint8_t *const *srcs, const size_t *pitches,
                     const std::function<int(const Slot &)> &download, unsigned long long *ticket)
{
    for (int i = 0; i < c->n; ++i)
        if (!srcs[i] || pitches[i] < (size_t)c->img[i].in_w * 3) {
            set_error("%s: invalid source %d", what, i);
            return SB_ERR_INVALID;
        }
    if (!pipe_ready(c)) SB_TRY(compositor_pipe_init(c));
    const unsigned long long t = c->submitted;
    const int slot = (int)(t % SB_PIPE_DEPTH);
    Slot &sl = c->slots[slot];
    // sources of this slot are free once the previous compute that read them has finished; on a slot's first use
    // that is whatever upload() / run() / sb_compositor_time() queued on the compute stream before this submit
    // (download() is synchronous, so the output buffers need no such guard)
    if (t < SB_PIPE_DEPTH) SB_CUDA(cudaEventRecord(sl.e_comp, c->stream));
    SB_CUDA(cudaStreamWaitEvent(c->h2d, sl.e_comp, 0));
    for (int i : c->warped) {
        const Image &im = c->img[i];
        SB_CUDA(sb_copy2d(sl.img[i].frame, (size_t)im.in_w * 3, srcs[i], pitches[i], (size_t)im.in_w * 3, im.in_h, cudaMemcpyHostToDevice, c->h2d));
    }
    // the repack (and resize) kernels follow the LAST copy (same stream): a kernel between two copies would leave the PCIe
    // link idle for its launch + run time, eight times per step
    SB_TRY(prepare_sources(c, sl, 0, c->n, c->h2d));
    SB_CUDA(cudaEventRecord(sl.e_h2d, c->h2d));
    SB_CUDA(cudaStreamWaitEvent(c->stream, sl.e_h2d, 0));
    // the output buffers of this slot (panorama or pasted parts) are free once their previous download has finished
    if (t >= SB_PIPE_DEPTH) SB_CUDA(cudaStreamWaitEvent(c->stream, sl.e_d2h, 0));
    SB_TRY(compositor_enqueue(c, false, slot));
    SB_CUDA(cudaEventRecord(sl.e_comp, c->stream));
    SB_CUDA(cudaStreamWaitEvent(c->d2h, sl.e_comp, 0));
    SB_TRY(download(sl));
    SB_CUDA(cudaEventRecord(sl.e_d2h, c->d2h));
    c->submitted = t + 1;
    if (ticket) *ticket = t;
    return SB_OK;
}

// blend: false when the rig's blend fields are unused (a timelapse compositor)
static bool valid_rig(const sb_rig *rig, bool blend = true)
{
    return rig && rig->n_images > 0 && rig->n_images <= SB_MAX_IMAGES && rig->src_w && rig->src_h && rig->K && rig->R &&
           rig->warp_type >= SB_WARP_SPHERICAL && rig->warp_type <= SB_WARP_TRANSVERSE_MERCATOR &&
           (!blend || (rig->blend_kind >= SB_BLEND_NO && rig->blend_kind <= SB_BLEND_MULTIBAND));
}

// what sb_compositor_create refuses before it builds anything
static bool valid_opts(const sb_rig *rig, const sb_compositor_opts &o)
{
    if (o.timelapse && o.timelapse != SB_TIMELAPSE_AS_IS && o.timelapse != SB_TIMELAPSE_CROP) {
        set_error("sb_compositor_create: unknown timelapse kind %d", o.timelapse);
        return false;
    }
    if (!valid_rig(rig, !o.timelapse) || o.world < 1 || o.rank < 0 || o.rank >= o.world || !o.in_w != !o.in_h ||
        (o.crop && (!o.crop->rect || !o.crop->corner || !o.crop->size))) {
        set_error("sb_compositor_create: invalid argument");
        return false;
    }
    if (o.timelapse && o.world > 1) {
        set_error("sb_compositor_create: invalid argument: a timelapse compositor runs on one GPU, not %d", o.world);
        return false;
    }
    return true;
}

// the entries that need a panorama, warped images, masks or a shard: a timelapse compositor has none of them
static bool refuse_timelapse(const sb_compositor *c, const char *what)
{
    if (!c || !c->timelapse) return false;
    set_error("%s: not available on a timelapse compositor, whose steps end in frames (sb_compositor_submit_timelapse)", what);
    return true;
}

extern "C" {

sb_compositor *sb_compositor_create(const sb_rig *rig, const sb_compositor_opts *opts)
{
    const sb_compositor_opts o = opts ? *opts : sb_compositor_opts{nullptr, nullptr, nullptr, 0, 1, 0};
    if (!valid_opts(rig, o)) return nullptr;
    sb_compositor *c = new sb_compositor;
    if (compositor_build(c, rig, o) != SB_OK) {
        compositor_free(c);
        return nullptr;
    }
    return c;
}

int sb_compositor_shard_info(const sb_compositor *c, int *first_image, int *n_local, int strip[2])
{
    if (!c) {
        set_error("sb_compositor_shard_info: null handle");
        return SB_ERR_INVALID;
    }
    if (first_image) *first_image = c->first;
    if (n_local) *n_local = c->count;
    if (strip) {
        strip[0] = 0;
        strip[1] = c->timelapse ? c->canvas.w : c->plan.roi.w;
        if (c->sharded) c->shard.strip(c->plan, &strip[0], &strip[1]);  // columns, or rows when sb_compositor_shard_axis() == 1
    }
    return SB_OK;
}

// Transport hooks: run the two halves of a sharded step separately and reach the slab buffers, so that a caller can
// move the slabs itself (tests do, with plain copies; sb_compositor_run uses the transport of ShardPlan).  Phase 0 is the
// warp and the step's loop 0, phase 1 its loop 1, both without the transport calls.
int sb_compositor_shard_phase(sb_compositor *c, int phase)
{
    if (refuse_timelapse(c, "sb_compositor_shard_phase")) return SB_ERR_STATE;
    if (!c || !c->sharded || phase < 0 || phase > 1) {
        set_error("sb_compositor_shard_phase: invalid argument");
        return SB_ERR_INVALID;
    }
    cudaStream_t s = c->stream;
    auto no_mark = [](const std::string &) -> int { return SB_OK; };
    if (phase == 0) {
        SB_TRY(launch_warp(warp_jobs(c, 0), (int)c->warped.size(), s));
        SB_TRY(shard_send_parts(c, false, s, no_mark));
    } else {
        SB_TRY(shard_finish_parts(c, c->slots[0].out, false, s, no_mark));
    }
    SB_CUDA(cudaStreamSynchronize(s));
    return SB_OK;
}

int sb_compositor_shard_axis(const sb_compositor *c) { return c && c->sharded ? c->shard.axis : 0; }

int sb_compositor_shard_slab(sb_compositor *c, int peer, int outgoing, void **dev_ptr, size_t *bytes)
{
    if (refuse_timelapse(c, "sb_compositor_shard_slab")) return SB_ERR_STATE;
    if (!c || !c->sharded || peer < 0 || peer >= c->shard.world || peer == c->shard.rank || !dev_ptr || !bytes) {
        set_error("sb_compositor_shard_slab: invalid argument");
        return SB_ERR_INVALID;
    }
    const PeerSlab &p = outgoing ? c->shard.send[peer] : c->shard.recv[peer];
    *dev_ptr = p.buf;
    *bytes = p.bytes;
    return SB_OK;
}

void sb_compositor_destroy(sb_compositor *c) { compositor_free(c); }

int sb_compositor_geometry(const sb_compositor *c, int *rects, int pano_roi[4], int *num_bands)
{
    if (!c) {
        set_error("sb_compositor_geometry: null handle");
        return SB_ERR_INVALID;
    }
    if (rects)
        for (int i = 0; i < c->n; ++i) {
            rects[4 * i] = c->img[i].rect.x;
            rects[4 * i + 1] = c->img[i].rect.y;
            rects[4 * i + 2] = c->img[i].rect.w;
            rects[4 * i + 3] = c->img[i].rect.h;
        }
    if (pano_roi) {
        const Rect &r = c->timelapse ? c->canvas : c->plan.roi;  // a timelapse: its canvas
        pano_roi[0] = r.x;
        pano_roi[1] = r.y;
        pano_roi[2] = r.w;
        pano_roi[3] = r.h;
    }
    if (num_bands) *num_bands = !c->timelapse && c->plan.kind == SB_BLEND_MULTIBAND ? c->plan.nb : -1;
    return SB_OK;
}

int sb_compositor_model_bytes(const sb_compositor *c, double *total_bytes, double *per_launch, int cap)
{
    if (!c) {
        set_error("sb_compositor_model_bytes: null handle");
        return SB_ERR_INVALID;
    }
    std::vector<double> v;
    v.push_back(c->warp_bytes);
    if (c->timelapse)
        v.push_back(c->paste_model);
    else
        for (const auto &kv : c->plan.launch_bytes()) v.push_back(kv.second);
    double tot = 0;
    for (double b : v) tot += b;
    if (total_bytes) *total_bytes = tot;
    if (per_launch)
        for (int i = 0; i < cap && i < (int)v.size(); ++i) per_launch[i] = v[i];
    return (int)v.size();
}

int sb_compositor_upload(sb_compositor *c, int i, const uint8_t *src, size_t pitch, int pinned)
{
    if (refuse_timelapse(c, "sb_compositor_upload")) return SB_ERR_STATE;
    if (!c || i < 0 || i >= c->n || !src || pitch < (size_t)c->img[i].in_w * 3) {
        set_error("sb_compositor_upload: invalid argument");
        return SB_ERR_INVALID;
    }
    if (!warped_here(c, i)) {
        set_error("sb_compositor_upload: image %d belongs to another rank (this rank owns %d..%d)", i, c->first, c->first + c->count - 1);
        return SB_ERR_INVALID;
    }
    const Image &im = c->img[i];
    SB_CUDA(sb_copy2d(c->slots[0].img[i].frame, (size_t)im.in_w * 3, src, pitch, (size_t)im.in_w * 3, im.in_h, cudaMemcpyHostToDevice, c->stream));
    SB_TRY(prepare_sources(c, c->slots[0], i, i + 1, c->stream));
    if (!pinned) SB_CUDA(cudaStreamSynchronize(c->stream));
    return SB_OK;
}

int sb_compositor_set_mask(sb_compositor *c, int i, const uint8_t *mask, size_t pitch)
{
    if (refuse_timelapse(c, "sb_compositor_set_mask")) return SB_ERR_STATE;  // the Timelapser ignores masks
    if (!c || i < 0 || i >= c->n || !mask || pitch < (size_t)c->img[i].rect.w || !warped_here(c, i)) {
        set_error("sb_compositor_set_mask: invalid argument (or an image of another rank)");
        return SB_ERR_INVALID;
    }
    // the blend mask of image i in warped coordinates (what stitcher.py:223-239 hands to Blender.feed); it replaces
    // the validity mask in the weight byte of the packed warped image from the next run on
    Image &im = c->img[i];
    const int w = im.rect.w, h = im.rect.h;
    if (!im.usermask) SB_TRY(dev_alloc((void **)&im.usermask, (size_t)w * h, c->stream));
    SB_CUDA(sb_copy2d(im.usermask, w, mask, pitch, w, h, cudaMemcpyHostToDevice, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    use_blend_mask(c, i, 0);
    return SB_OK;
}

int sb_compositor_set_seam_mask(sb_compositor *c, int i, const uint8_t *seam, size_t seam_pitch, int sw, int sh)
{
    if (refuse_timelapse(c, "sb_compositor_set_seam_mask")) return SB_ERR_STATE;
    if (!c || i < 0 || i >= c->n || !seam || sw <= 0 || sh <= 0 || seam_pitch < (size_t)sw || !warped_here(c, i)) {
        set_error("sb_compositor_set_seam_mask: invalid argument (or an image of another rank)");
        return SB_ERR_INVALID;
    }
    // SeamFinder.resize(seam_mask, warped mask) (seam_finder.py:38-43, stitcher.py:223-225) without the host round
    // trip: the LOW-resolution seam mask is dilated and resized on the device; the AND with the warped validity mask
    // happens in the warp kernel, which computes that mask anyway
    Image &im = c->img[i];
    const int w = im.rect.w, h = im.rect.h;
    if (!im.usermask) SB_TRY(dev_alloc((void **)&im.usermask, (size_t)w * h, c->stream));
    SB_TRY(seam_resize_device(seam, seam_pitch, sw, sh, nullptr, 0, im.usermask, w, w, h, c->stream));
    use_blend_mask(c, i, 1);
    return SB_OK;
}

int sb_compositor_set_gain(sb_compositor *c, int i, const float *gain_map, int gw, int gh, int gc, const double *gain_scalar)
{
    if (!c || i < 0 || i >= c->n || (!warped_here(c, i) && !c->timelapse) || (gain_map && gain_scalar) ||
        (gain_map && (gw <= 0 || gh <= 0 || (gc != 1 && gc != 3)))) {
        set_error("sb_compositor_set_gain: invalid argument (or an image of another rank)");
        return SB_ERR_INVALID;
    }
    if (!warped_here(c, i)) return SB_OK;  // off the timelapse canvas: nothing of it is shown
    // ExposureErrorCompensator.apply(i, corner, warped image, mask) (exposure_error_compensator.py:43-45,
    // stitcher.py:219-221) fused into the warp's epilogue: the warped image never exists uncompensated
    SB_CUDA(cudaStreamSynchronize(c->stream));  // the previous run may still read the old gain buffers
    drop_graphs(c);  // before the upload, which frees the buffers they read
    Image &im = c->img[i];
    const Rect &r = im.rect;
    if (c->timelapse) {
        // only P_i is warped, but the gain map is resized to the whole fed image: the taps at P_i's place in it
        const Rect &p = im.part;
        const int sub[4] = {p.x - r.x, p.y - r.y, p.w, p.h};
        return gain_upload(&im.job, &im.gain, r.w, r.h, gain_map, gw, gh, gc, gain_scalar, c->stream, sub);
    }
    return gain_upload(&im.job, &im.gain, r.w, r.h, gain_map, gw, gh, gc, gain_scalar, c->stream);
}

int sb_compositor_run(sb_compositor *c)
{
    if (!c) {
        set_error("sb_compositor_run: null handle");
        return SB_ERR_INVALID;
    }
    if (refuse_timelapse(c, "sb_compositor_run")) return SB_ERR_STATE;
    return compositor_enqueue(c, false);
}

int sb_compositor_sync(sb_compositor *c)
{
    if (!c) return SB_ERR_INVALID;
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return SB_OK;
}

int sb_compositor_download(sb_compositor *c, uint8_t *dst, size_t dst_pitch, uint8_t *dst_mask, size_t mask_pitch)
{
    if (refuse_timelapse(c, "sb_compositor_download")) return SB_ERR_STATE;
    if (!c || (dst && dst_pitch < (size_t)c->slots[0].out.w * 3) || (dst_mask && mask_pitch < (size_t)c->slots[0].out.w)) {
        set_error("sb_compositor_download: invalid argument");
        return SB_ERR_INVALID;
    }
    SB_TRY(download_out(c->slots[0].out, dst, dst_pitch, dst_mask, mask_pitch, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return SB_OK;
}

// Pipelined end-to-end step: the D2H of the panorama ends it (pipe_step).
int sb_compositor_submit(sb_compositor *c, const uint8_t *const *srcs, const size_t *pitches, uint8_t *dst, size_t dst_pitch,
                         uint8_t *dst_mask, size_t mask_pitch, unsigned long long *ticket)
{
    if (refuse_timelapse(c, "sb_compositor_submit")) return SB_ERR_STATE;
    if (!c || !srcs || !pitches || (dst && dst_pitch < (size_t)c->slots[0].out.w * 3) || (dst_mask && mask_pitch < (size_t)c->slots[0].out.w)) {
        set_error("sb_compositor_submit: invalid argument");
        return SB_ERR_INVALID;
    }
    if (c->sharded) {
        set_error("sb_compositor_submit: the pipelined path is single-GPU; use upload / run / download on a sharded compositor");
        return SB_ERR_STATE;
    }
    auto download = [&](const Slot &sl) { return download_out(sl.out, dst, dst_pitch, dst_mask, mask_pitch, c->d2h); };
    return pipe_step(c, "sb_compositor_submit", srcs, pitches, download, ticket);
}

int sb_compositor_wait(sb_compositor *c, unsigned long long ticket)
{
    if (!c || c->n_slots < SB_PIPE_DEPTH || ticket >= c->submitted || ticket + SB_PIPE_DEPTH < c->submitted) {
        set_error("sb_compositor_wait: ticket %llu is not in flight", ticket);
        return SB_ERR_STATE;
    }
    SB_CUDA(cudaEventSynchronize(c->slots[ticket % SB_PIPE_DEPTH].e_d2h));
    return SB_OK;
}

// Pipelined timelapse step: H2D of the images on the canvas, warp + paste, then one 2D copy per image from its pasted part
// into its frame of this slot at P_i (the rest of every frame stays zero).  The ticket works with sb_compositor_wait.
int sb_compositor_submit_timelapse(sb_compositor *c, const uint8_t *const *srcs, const size_t *pitches, unsigned long long *ticket)
{
    if (!c || !srcs || !pitches) {
        set_error("sb_compositor_submit_timelapse: invalid argument");
        return SB_ERR_INVALID;
    }
    if (!c->timelapse) {
        set_error("sb_compositor_submit_timelapse: not a timelapse compositor (sb_compositor_opts.timelapse)");
        return SB_ERR_STATE;
    }
    auto download = [c](const Slot &sl) -> int {
        const Rect &cv = c->canvas;
        const size_t fpitch = (size_t)cv.w * 3, fbytes = fpitch * cv.h;
        for (int i : c->warped) {
            const Rect &p = c->img[i].part;
            uint8_t *dst = sl.frames + fbytes * i + (size_t)(p.y - cv.y) * fpitch + (size_t)(p.x - cv.x) * 3;
            SB_CUDA(sb_copy2d(dst, fpitch, sl.paste + c->img[i].paste_off, (size_t)p.w * 3, (size_t)p.w * 3, p.h, cudaMemcpyDeviceToHost, c->d2h));
        }
        return SB_OK;
    };
    return pipe_step(c, "sb_compositor_submit_timelapse", srcs, pitches, download, ticket);
}

int sb_compositor_timelapse_frame(const sb_compositor *c, unsigned long long ticket, int i, const uint8_t **frame, size_t *pitch)
{
    if (!c || i < 0 || i >= c->n || !frame || !pitch) {
        set_error("sb_compositor_timelapse_frame: invalid argument");
        return SB_ERR_INVALID;
    }
    if (!c->timelapse || !pipe_ready(c) || ticket >= c->submitted || ticket + SB_PIPE_DEPTH < c->submitted) {
        set_error("sb_compositor_timelapse_frame: ticket %llu is not in flight on a timelapse compositor", ticket);
        return SB_ERR_STATE;
    }
    *pitch = (size_t)c->canvas.w * 3;
    *frame = c->slots[ticket % SB_PIPE_DEPTH].frames + *pitch * c->canvas.h * i;
    return SB_OK;
}

int sb_compositor_download_warped(sb_compositor *c, int i, uint8_t *dst, size_t dst_pitch, uint8_t *dst_mask, size_t mask_pitch)
{
    if (refuse_timelapse(c, "sb_compositor_download_warped")) return SB_ERR_STATE;
    if (!c || i < 0 || i >= c->n || !warped_here(c, i)) {
        set_error("sb_compositor_download_warped: invalid argument (or an image of another rank)");
        return SB_ERR_INVALID;
    }
    const int w = c->img[i].rect.w, h = c->img[i].rect.h;
    const size_t wp = (size_t)rgbm_pitch_of(w);
    std::vector<uint32_t> tmp(wp * h);
    SB_CUDA(cudaMemcpyAsync(tmp.data(), c->img[i].rgbm, tmp.size() * 4, cudaMemcpyDeviceToHost, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            const uint32_t p = tmp[(size_t)y * wp + x];
            if (dst) {
                uint8_t *d = dst + (size_t)y * dst_pitch + (size_t)x * 3;
                d[0] = p & 255;
                d[1] = (p >> 8) & 255;
                d[2] = (p >> 16) & 255;
            }
            if (dst_mask) dst_mask[(size_t)y * mask_pitch + x] = (uint8_t)(p >> 24);
        }
    return SB_OK;
}

// Throughput with several batches in flight: `iters` steps dealt round-robin to n compositors of the same rig (each
// has its own stream and buffers, so the small latency-bound kernels of one step overlap the large kernels of
// another).  One start event; every stream waits for it; the time is up to the LAST stream's end event.
int sb_compositor_time_multi(sb_compositor *const *cs, int n, int iters, float *ms_total)
{
    if (!cs || n < 1 || n > 8 || iters <= 0 || !ms_total) {
        set_error("sb_compositor_time_multi: invalid argument");
        return SB_ERR_INVALID;
    }
    for (int k = 0; k < n; ++k)
        if (refuse_timelapse(cs[k], "sb_compositor_time_multi")) return SB_ERR_STATE;
    for (int k = 0; k < n; ++k)
        if (!cs[k] || cs[k]->sharded) {
            set_error("sb_compositor_time_multi: null or sharded compositor");
            return SB_ERR_INVALID;
        }
    cudaEvent_t start = nullptr, ends[8] = {};
    SB_CUDA(cudaEventCreate(&start));
    for (int k = 0; k < n; ++k) SB_CUDA(cudaEventCreate(&ends[k]));
    SB_CUDA(cudaEventRecord(start, cs[0]->stream));
    for (int k = 1; k < n; ++k) SB_CUDA(cudaStreamWaitEvent(cs[k]->stream, start, 0));
    int rc = SB_OK;
    for (int it = 0; it < iters && rc == SB_OK; ++it) rc = compositor_enqueue(cs[it % n], false);
    float worst = 0.f;
    for (int k = 0; k < n; ++k) {
        if (cudaEventRecord(ends[k], cs[k]->stream) != cudaSuccess || cudaEventSynchronize(ends[k]) != cudaSuccess) rc = rc == SB_OK ? SB_ERR_CUDA : rc;
        float t = 0.f;
        if (rc == SB_OK && cudaEventElapsedTime(&t, start, ends[k]) == cudaSuccess) worst = t > worst ? t : worst;
    }
    (void)cudaEventDestroy(start);
    for (int k = 0; k < n; ++k) (void)cudaEventDestroy(ends[k]);
    if (rc != SB_OK && rc == SB_ERR_CUDA) set_error("sb_compositor_time_multi: CUDA failure while timing");
    *ms_total = worst;
    return rc;
}

int sb_compositor_time(sb_compositor *c, int iters, int flush_l2, float *ms_total)
{
    if (!c || iters <= 0 || !ms_total) {
        set_error("sb_compositor_time: invalid argument");
        return SB_ERR_INVALID;
    }
    cudaStream_t s = c->stream;
    if (flush_l2 && !c->flush_buf) {
        c->flush_bytes = (size_t)128 << 20;  // more than 2x the 50 MB L2 of an H100
        SB_TRY(dev_alloc(&c->flush_buf, c->flush_bytes, s));
    }
    float total = 0.f;
    // pass 1: whole steps exactly as sb_compositor_run issues them (one graph launch), one event pair per step
    // (the host enqueues ahead of the device: no host synchronisation between steps; with flush_l2 the flush
    // kernel runs between a step's end event and the next step's start event)
    while ((int)c->tev.size() < 2 * iters) {
        cudaEvent_t e;
        SB_CUDA(cudaEventCreate(&e));
        c->tev.push_back(e);
    }
    for (int it = 0; it < iters; ++it) {
        if (flush_l2) SB_TRY(launch_flush_l2(c->flush_buf, c->flush_bytes, s));
        if (flush_l2 || it == 0) SB_CUDA(cudaEventRecord(c->tev[2 * it], s));
        SB_TRY(compositor_enqueue(c, false));
        if (flush_l2 || it == iters - 1) SB_CUDA(cudaEventRecord(c->tev[2 * it + 1], s));
    }
    SB_CUDA(cudaStreamSynchronize(s));
    if (flush_l2) {
        for (int it = 0; it < iters; ++it) {
            float t = 0;
            SB_CUDA(cudaEventElapsedTime(&t, c->tev[2 * it], c->tev[2 * it + 1]));
            total += t;
        }
    } else {
        SB_CUDA(cudaEventElapsedTime(&total, c->tev[0], c->tev[2 * (iters - 1) + 1]));
    }
    *ms_total = total;
    // pass 2: per-kernel breakdown (individual launches with an event after each), a few iterations
    iters = iters < 5 ? iters : 5;
    c->launch_ms.clear();
    for (int it = 0; it < iters; ++it) {
        if (flush_l2) SB_TRY(launch_flush_l2(c->flush_buf, c->flush_bytes, s));
        SB_TRY(compositor_enqueue(c, true));
        const size_t nl = c->launch_names.size();
        SB_CUDA(cudaEventSynchronize(c->ev[nl]));
        if (c->launch_ms.size() != nl) c->launch_ms.assign(nl, 0.f);
        for (size_t k = 0; k < nl; ++k) {
            float t = 0;
            SB_CUDA(cudaEventElapsedTime(&t, c->ev[k], c->ev[k + 1]));
            c->launch_ms[k] += t;
        }
    }
    for (float &v : c->launch_ms) v /= (float)iters;
    return SB_OK;
}

int sb_compositor_stage_times(sb_compositor *c, const char **names, float *ms, int cap)
{
    if (!c) return 0;
    int k = (int)std::min<size_t>((size_t)cap, c->launch_ms.size());
    for (int i = 0; i < k; ++i) {
        if (names) names[i] = c->launch_names[i].c_str();
        if (ms) ms[i] = c->launch_ms[i];
    }
    return k;
}

}  // extern "C"
