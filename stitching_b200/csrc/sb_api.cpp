// sb_api.cpp -- the C ABI (include/stitch_b200.h): Warper and Blender entry points with host buffers.  Each of them checks
// its arguments, stages the host buffers on the device, runs the device core and finishes (sb::Staging).
#include <cstring>
#include <mutex>
#include <vector>

#include "sb_plan.h"

using namespace sb;

static bool valid_warp_type(int t) { return t >= SB_WARP_SPHERICAL && t <= SB_WARP_TRANSVERSE_MERCATOR; }

struct sb_devimg {
    uint8_t *p;
    int w, h, ch;
};

// The reference asks for the same roi several times per image -- warp_roi, then warp (image), then warp (mask), each of
// which runs detectResultRoi again (warper.py:43-82) -- and for eleven of the projections that is a pass over EVERY source
// pixel.  The result depends on nothing but the arguments, so the last few are remembered (host memory, a few hundred bytes).
namespace {
struct RoiKey {
    int type, w, h;
    float scale, K[9], R[9];
};
struct RoiEntry {
    RoiKey key;
    int rect[4];
};
std::mutex g_roi_mutex;
std::vector<RoiEntry> g_roi_cache;  // most recent last
constexpr size_t ROI_CACHE_ENTRIES = 64;

void cached_roi(const Projector &p, int warp_type, float scale, const float K[9], const float R[9], int src_w, int src_h, int rect[4])
{
    RoiKey key;
    std::memset(&key, 0, sizeof key);
    key.type = warp_type;
    key.w = src_w;
    key.h = src_h;
    key.scale = scale;
    std::memcpy(key.K, K, sizeof key.K);
    std::memcpy(key.R, R, sizeof key.R);
    {
        std::lock_guard<std::mutex> lock(g_roi_mutex);
        for (size_t i = g_roi_cache.size(); i-- > 0;)
            if (!std::memcmp(&g_roi_cache[i].key, &key, sizeof key)) {  // bit patterns: -0.0f and NaNs simply miss
                std::memcpy(rect, g_roi_cache[i].rect, sizeof g_roi_cache[i].rect);
                return;
            }
    }
    projector_roi(p, src_w, src_h, rect);
    RoiEntry e;
    e.key = key;
    std::memcpy(e.rect, rect, sizeof e.rect);
    std::lock_guard<std::mutex> lock(g_roi_mutex);
    if (g_roi_cache.size() >= ROI_CACHE_ENTRIES) g_roi_cache.erase(g_roi_cache.begin());
    g_roi_cache.push_back(e);
}
}  // namespace

extern "C" {

int sb_warp_roi(int warp_type, float scale, const float K[9], const float R[9], int src_w, int src_h, int out_rect[4])
{
    if (!valid_warp_type(warp_type) || !K || !R || !out_rect || src_w <= 0 || src_h <= 0) {
        set_error("sb_warp_roi: invalid argument");
        return SB_ERR_INVALID;
    }
    Projector p;
    projector_setup(p, warp_type, scale, K, R);
    cached_roi(p, warp_type, scale, K, R, src_w, src_h, out_rect);
    return SB_OK;
}

static int warp_impl(int warp_type, float scale, const float K[9], const float R[9], const uint8_t *src, int src_w, int src_h,
                     size_t src_pitch, uint8_t *dst_img, size_t dst_pitch, uint8_t *dst_mask, size_t mask_pitch, int out_rect[4],
                     sb_devimg **keep_img, sb_devimg **keep_mask)
{
    if (keep_img) *keep_img = nullptr;
    if (keep_mask) *keep_mask = nullptr;
    if (!valid_warp_type(warp_type) || !K || !R || !out_rect || src_w <= 0 || src_h <= 0 || (dst_img && !src) ||
        (src && src_pitch < (size_t)src_w * 3)) {
        set_error("sb_warp: invalid argument");
        return SB_ERR_INVALID;
    }
    Projector p;
    projector_setup(p, warp_type, scale, K, R);
    int rect[4];
    cached_roi(p, warp_type, scale, K, R, src_w, src_h, rect);
    std::memcpy(out_rect, rect, sizeof rect);
    if (!dst_img && !dst_mask) return SB_OK;
    const int w = rect[2], h = rect[3];
    if (w <= 0 || h <= 0 || (long long)w * h > (1ll << 31)) {
        set_error("sb_warp: degenerate result roi %dx%d", w, h);
        return SB_ERR_INVALID;
    }
    if ((dst_img && dst_pitch < (size_t)w * 3) || (dst_mask && mask_pitch < (size_t)w)) {
        set_error("sb_warp: destination pitch too small for roi width %d", w);
        return SB_ERR_INVALID;
    }
    // cv::remap asserts that both images are narrower and lower than SHRT_MAX (the warp of the image and the warp of the
    // mask alike); warpRoi does not, so the roi-only call above still answers
    if (src_w >= SB_MAX_WARP_SIDE || src_h >= SB_MAX_WARP_SIDE || w >= SB_MAX_WARP_SIDE || h >= SB_MAX_WARP_SIDE) {
        set_error("sb_warp: source %dx%d or result %dx%d has a side of %d px or more, which cv::remap refuses", src_w, src_h, w, h,
                  SB_MAX_WARP_SIDE);
        return SB_ERR_INVALID;
    }
    SB_TRY(ensure_device());
    std::vector<float> host_tab;
    Staging st(default_stream());
    cudaStream_t s = st.stream();
    WarpJob job;
    float *tab = st.tmp<float>(warp_table_floats(w, h));
    st.run([&] { return make_warp_job(p, rect, src_w, src_h, tab, &job, s, host_tab); });
    if (projector_needs_maps(p)) {
        float *maps = st.tmp<float>((size_t)2 * w * h);
        st.run([&] { return warp_maps_upload(p, rect, maps, &job, s); });
    }
    // the kept image and mask survive the call inside their handles
    const bool keep_i = dst_img && keep_img, keep_m = dst_mask && keep_mask;
    uint8_t *d_img = nullptr, *d_mask = nullptr;
    if (dst_img) {
        uint8_t *d_src = st.tmp<uint8_t>((size_t)src_w * 3 * src_h + SB_SRC_PAD);
        d_img = keep_i ? st.keep<uint8_t>((size_t)w * 3 * h) : st.tmp<uint8_t>((size_t)w * 3 * h);
        st.copy(d_src, (size_t)src_w * 3, src, src_pitch, (size_t)src_w * 3, src_h, cudaMemcpyHostToDevice);
        job.src = d_src;
        job.spitch = (long long)src_w * 3;
        job.dst_rgb = d_img;
        job.dst_pitch = (long long)w * 3;
    }
    if (dst_mask) {
        d_mask = keep_m ? st.keep<uint8_t>((size_t)w * h) : st.tmp<uint8_t>((size_t)w * h);
        job.dst_mask = d_mask;
        job.mask_pitch = w;
    }
    st.run([&] { return launch_warp(&job, 1, s); });
    if (dst_img) st.down(dst_img, dst_pitch, d_img, (size_t)w * 3, (size_t)w * 3, h);
    if (dst_mask) st.down(dst_mask, mask_pitch, d_mask, w, w, h);
    SB_TRY(st.finish());
    if (keep_i) *keep_img = new sb_devimg{d_img, w, h, 3};
    if (keep_m) *keep_mask = new sb_devimg{d_mask, w, h, 1};
    return SB_OK;
}

int sb_warp(int warp_type, float scale, const float K[9], const float R[9], const uint8_t *src, int src_w, int src_h,
            size_t src_pitch, uint8_t *dst_img, size_t dst_pitch, uint8_t *dst_mask, size_t mask_pitch, int out_rect[4])
{
    return warp_impl(warp_type, scale, K, R, src, src_w, src_h, src_pitch, dst_img, dst_pitch, dst_mask, mask_pitch, out_rect, nullptr, nullptr);
}

int sb_warp_keep(int warp_type, float scale, const float K[9], const float R[9], const uint8_t *src, int src_w, int src_h,
                 size_t src_pitch, uint8_t *dst_img, size_t dst_pitch, uint8_t *dst_mask, size_t mask_pitch, int out_rect[4],
                 sb_devimg **keep_img, sb_devimg **keep_mask)
{
    return warp_impl(warp_type, scale, K, R, src, src_w, src_h, src_pitch, dst_img, dst_pitch, dst_mask, mask_pitch, out_rect, keep_img, keep_mask);
}

void sb_devimg_release(sb_devimg *d)
{
    if (!d) return;
    dev_free(d->p, default_stream());
    delete d;
}

int sb_devimg_info(const sb_devimg *d, int *w, int *h, int *channels)
{
    if (!d) {
        set_error("sb_devimg_info: null handle");
        return SB_ERR_INVALID;
    }
    if (w) *w = d->w;
    if (h) *h = d->h;
    if (channels) *channels = d->ch;
    return SB_OK;
}

}  // extern "C"

static bool valid_gain_args(const float *gain_map, int gw, int gh, int gc, const double *gain_scalar)
{
    if (gain_map && gain_scalar) return false;
    if (gain_map && (gw <= 0 || gh <= 0 || (gc != 1 && gc != 3))) return false;
    return true;
}

// ExposureErrorCompensator.apply on a device rectangle (pitch in bytes), then its copy to `host` when one is given
static int gain_apply(Staging &st, uint8_t *img, long long pitch, int w, int h, uint8_t *host, size_t host_pitch, const float *gain_map,
                      int gw, int gh, int gc, const double *gain_scalar)
{
    WarpJob job;
    std::memset(&job, 0, sizeof job);
    GainData gd;
    st.run([&] { return gain_upload(&job, &gd, w, h, gain_map, gw, gh, gc, gain_scalar, st.stream()); });
    st.run([&] { return launch_gain_apply(img, pitch, w, h, job, st.stream()); });
    if (host) st.down(host, host_pitch, img, (size_t)pitch, (size_t)w * 3, h);
    const int rc = st.finish();
    gain_free(&gd, st.stream());
    return rc;
}

extern "C" {

int sb_gain_apply(uint8_t *img, size_t pitch, int w, int h, const float *gain_map, int gw, int gh, int gc, const double *gain_scalar)
{
    if (!img || w <= 0 || h <= 0 || pitch < (size_t)w * 3 || !valid_gain_args(gain_map, gw, gh, gc, gain_scalar)) {
        set_error("sb_gain_apply: invalid argument");
        return SB_ERR_INVALID;
    }
    if (!gain_map && !gain_scalar) return SB_OK;  // compensator "no": identity
    SB_TRY(ensure_device());
    Staging st(default_stream());
    uint8_t *d_img = st.up<uint8_t>(img, pitch, (size_t)w * 3, h);
    return gain_apply(st, d_img, (long long)w * 3, w, h, img, pitch, gain_map, gw, gh, gc, gain_scalar);
}

int sb_gain_apply_dev(sb_devimg *img, int x, int y, int w, int h, uint8_t *host, size_t host_pitch, const float *gain_map, int gw, int gh,
                      int gc, const double *gain_scalar)
{
    if (!img || img->ch != 3 || x < 0 || y < 0 || w <= 0 || h <= 0 || x + w > img->w || y + h > img->h || (host && host_pitch < (size_t)w * 3) ||
        !valid_gain_args(gain_map, gw, gh, gc, gain_scalar)) {
        set_error("sb_gain_apply_dev: invalid argument");
        return SB_ERR_INVALID;
    }
    if (!gain_map && !gain_scalar) return SB_OK;  // compensator "no": identity (host and device copies stay as they are)
    SB_TRY(ensure_device());
    Staging st(default_stream());
    uint8_t *view = img->p + ((size_t)y * img->w + x) * 3;
    return gain_apply(st, view, (long long)img->w * 3, w, h, host, host_pitch, gain_map, gw, gh, gc, gain_scalar);
}

int sb_timelapse_frame(const void *img, int is_s16, size_t pitch, const sb_devimg *dev, int dev_x, int dev_y, int w, int h, int tlx, int tly,
                       const int roi[4], uint8_t *dst, size_t dst_pitch)
{
    const size_t px = is_s16 ? 6 : 3;
    if ((!img && !dev) || !roi || !dst || w <= 0 || h <= 0 || roi[2] <= 0 || roi[3] <= 0 || dst_pitch < (size_t)roi[2] * 3 ||
        (long long)roi[2] * roi[3] > (1ll << 31) || (!dev && pitch < (size_t)w * px) ||
        (dev && (dev->ch != 3 || dev_x < 0 || dev_y < 0 || dev_x + w > dev->w || dev_y + h > dev->h))) {
        set_error("sb_timelapse_frame: invalid argument");
        return SB_ERR_INVALID;
    }
    SB_TRY(ensure_device());
    Staging st(default_stream());
    const int cw = roi[2], ch = roi[3];
    uint8_t *d_dst = st.tmp<uint8_t>((size_t)cw * 3 * ch);
    // a device source is uint8; from the host, only the rows / columns that land on the canvas travel.  spitch: bytes of
    // a uint8 row, elements of an int16 row
    const bool s16 = is_s16 && !dev;
    const uint8_t *src = dev ? dev->p + ((size_t)dev_y * dev->w + dev_x) * 3 : st.up<uint8_t>(img, pitch, (size_t)w * px, h);
    const long long spitch = dev ? (long long)dev->w * 3 : (long long)w * 3;
    st.run([&] {
        return launch_timelapse_frame(s16 ? nullptr : src, s16 ? (const int16_t *)src : nullptr, spitch, w, h, tlx - roi[0], tly - roi[1],
                                      d_dst, (long long)cw * 3, cw, ch, st.stream());
    });
    st.down(dst, dst_pitch, d_dst, (size_t)cw * 3, (size_t)cw * 3, ch);
    return st.finish();
}

int sb_resize_exact(const uint8_t *src, size_t src_pitch, int sw, int sh, int channels, uint8_t *dst, size_t dst_pitch, int dw, int dh)
{
    if (!src || !dst || sw <= 0 || sh <= 0 || dw <= 0 || dh <= 0 || (channels != 1 && channels != 3) ||
        src_pitch < (size_t)sw * channels || dst_pitch < (size_t)dw * channels || (long long)sw * sh * channels > (1ll << 31) ||
        (long long)dw * dh * channels > (1ll << 31)) {
        set_error("sb_resize_exact: invalid argument");
        return SB_ERR_INVALID;
    }
    SB_TRY(ensure_device());
    std::vector<int> tx((size_t)3 * dw), ty((size_t)3 * dh);
    resize_exact_taps(sw, dw, tx.data());
    resize_exact_taps(sh, dh, ty.data());
    Staging st(default_stream());
    const size_t srow = (size_t)sw * channels, drow = (size_t)dw * channels;
    const uint8_t *d_src = st.up<uint8_t>(src, src_pitch, srow, sh);
    uint8_t *d_dst = st.tmp<uint8_t>(drow * dh);
    const int *d_tx = st.up(tx), *d_ty = st.up(ty);
    st.run([&] { return launch_resize_exact(d_src, (long long)srow, channels, d_tx, d_ty, d_dst, (long long)drow, dw, dh, st.stream()); });
    st.down(dst, dst_pitch, d_dst, drow, drow, dh);
    return st.finish();
}

int sb_seam_resize(const uint8_t *seam, size_t seam_pitch, int sw, int sh, const uint8_t *mask, size_t mask_pitch, int w, int h,
                   uint8_t *dst, size_t dst_pitch)
{
    if (!seam || !mask || !dst || sw <= 0 || sh <= 0 || w <= 0 || h <= 0 || seam_pitch < (size_t)sw || mask_pitch < (size_t)w ||
        dst_pitch < (size_t)w || (long long)w * h > (1ll << 31) || (long long)sw * sh > (1ll << 31)) {
        set_error("sb_seam_resize: invalid argument");
        return SB_ERR_INVALID;
    }
    SB_TRY(ensure_device());
    Staging st(default_stream());
    const uint8_t *d_mask = st.up<uint8_t>(mask, mask_pitch, w, h);
    uint8_t *d_dst = st.tmp<uint8_t>((size_t)w * h);
    st.run([&] { return seam_resize_device(seam, seam_pitch, sw, sh, d_mask, w, d_dst, w, w, h, st.stream()); });
    st.down(dst, dst_pitch, d_dst, w, w, h);
    return st.finish();
}

// -------------------------------------------------------------------------------------------------
// Blender
// -------------------------------------------------------------------------------------------------
struct sb_blender {
    int kind;
    int num_bands;
    float sharpness;
    bool prepared = false;
    BlendPlan plan;
    std::vector<void *> level0;  // device buffers of the recorded feeds
};

sb_blender *sb_blender_create(int kind, int num_bands, float sharpness)
{
    if (kind < SB_BLEND_NO || kind > SB_BLEND_MULTIBAND) {
        set_error("sb_blender_create: unknown kind %d", kind);
        return nullptr;
    }
    sb_blender *b = new sb_blender;
    b->kind = kind;
    b->num_bands = num_bands;
    b->sharpness = sharpness;
    return b;
}

static void blender_drop_feeds(sb_blender *b)
{
    cudaStream_t s = default_stream();
    for (void *p : b->level0) dev_free(p, s);
    b->level0.clear();
    b->plan.release(s);
    b->plan.imgs.clear();
}

void sb_blender_destroy(sb_blender *b)
{
    if (!b) return;
    blender_drop_feeds(b);
    delete b;
}

int sb_blender_prepare(sb_blender *b, int x, int y, int w, int h)
{
    if (!b) {
        set_error("sb_blender_prepare: null handle");
        return SB_ERR_INVALID;
    }
    blender_drop_feeds(b);
    b->prepared = false;
    SB_TRY(b->plan.set_geometry(b->kind, b->num_bands, b->sharpness, Rect{x, y, w, h}));
    b->prepared = true;
    return SB_OK;
}

int sb_blender_num_bands(const sb_blender *b) { return b ? b->plan.nb : -1; }

// one recorded feed: geometry first (host only, so that an out-of-roi feed fails before any device work), then the level-0
// data on the device.  The image comes from the host (img) or from a device rectangle (dimg, dimg_pitch); likewise the mask.
// A feed that fails leaves the blender as it was.
static int blender_feed_impl(sb_blender *b, const void *img, int img_is_s16, size_t img_pitch, const uint8_t *dimg, size_t dimg_pitch,
                             const uint8_t *mask, size_t mask_pitch, const uint8_t *dmask, size_t dmask_pitch, int w, int h, int tl_x, int tl_y)
{
    FeedDesc f;
    std::memset(&f, 0, sizeof f);
    f.w = w; f.h = h; f.tlx = tl_x; f.tly = tl_y;
    SB_TRY(b->plan.add_feed(f));
    FeedImage &im = b->plan.imgs.back();
    int rc = ensure_device();
    if (rc == SB_OK) {
        Staging st(default_stream());
        cudaStream_t s = st.stream();
        const size_t px_bytes = img_is_s16 ? 6 : 3;
        const bool host_mask = !dmask;
        // host images and masks are staged into buffers the blender keeps: from here on both sources are on the device
        if (host_mask) {
            uint8_t *d = st.keep<uint8_t>((size_t)w * h);
            st.copy(d, w, mask, mask_pitch, w, h, cudaMemcpyHostToDevice);
            dmask = d;
            dmask_pitch = w;
        }
        if (!dimg) {
            uint8_t *d = st.keep<uint8_t>((size_t)w * h * px_bytes);
            st.copy(d, (size_t)w * px_bytes, img, img_pitch, (size_t)w * px_bytes, h, cudaMemcpyHostToDevice);
            dimg = d;
            dimg_pitch = (size_t)w * px_bytes;
        }
        if (img_is_s16) {
            if (!host_mask) {  // the generic layout keeps a pointer to the mask: it has to outlive this call
                uint8_t *d = st.keep<uint8_t>((size_t)w * h);
                st.copy(d, w, dmask, dmask_pitch, w, h, cudaMemcpyDeviceToDevice);
                dmask = d;
                dmask_pitch = w;
            }
            im.s16 = (const int16_t *)dimg;
            im.s16_pitch = (long long)w * 3;
            im.mask = dmask;
            im.mask_pitch = (long long)dmask_pitch;
        } else {
            const int rp = (w + 3) & ~3;  // 16-byte rows: the tile kernels stage windows of this buffer with 16-byte copies
            uint32_t *d_rgbm = st.keep<uint32_t>((size_t)rp * h);
            if (rp != w)  // zero row padding = weight 0
                st.run([&]() -> int {
                    SB_CUDA(cudaMemsetAsync(d_rgbm, 0, (size_t)rp * h * 4, s));
                    return SB_OK;
                });
            st.run([&] { return launch_pack_rgbm(dimg, (long long)dimg_pitch, dmask, (long long)dmask_pitch, d_rgbm, rp, w, h, s); });
            im.rgbm = d_rgbm;
            im.rgbm_pitch = rp;
        }
        // the caller's buffers (and device twins) may change as soon as we return
        rc = st.finish();
        if (rc == SB_OK) b->level0.insert(b->level0.end(), st.kept().begin(), st.kept().end());
    }
    if (rc != SB_OK) b->plan.imgs.pop_back();
    return rc;
}

int sb_blender_feed(sb_blender *b, const void *img, int img_is_s16, size_t img_pitch, const uint8_t *mask, size_t mask_pitch,
                    int w, int h, int tl_x, int tl_y)
{
    if (!b || !img || !mask || w <= 0 || h <= 0) {
        set_error("sb_blender_feed: invalid argument");
        return SB_ERR_INVALID;
    }
    if (!b->prepared) {
        set_error("sb_blender_feed: prepare() has not been called");
        return SB_ERR_STATE;
    }
    const size_t px_bytes = img_is_s16 ? 6 : 3;
    if (img_pitch < (size_t)w * px_bytes || mask_pitch < (size_t)w) {
        set_error("sb_blender_feed: pitch smaller than a row");
        return SB_ERR_INVALID;
    }
    return blender_feed_impl(b, img, img_is_s16, img_pitch, nullptr, 0, mask, mask_pitch, nullptr, 0, w, h, tl_x, tl_y);
}

int sb_blender_feed_dev(sb_blender *b, const sb_devimg *img, int ix, int iy, const sb_devimg *mask_dev, int mx, int my,
                        const uint8_t *mask_host, size_t mask_pitch, int w, int h, int tl_x, int tl_y)
{
    if (!b || !img || img->ch != 3 || w <= 0 || h <= 0 || ix < 0 || iy < 0 || ix + w > img->w || iy + h > img->h ||
        (!mask_dev && (!mask_host || mask_pitch < (size_t)w)) ||
        (mask_dev && (mask_dev->ch != 1 || mx < 0 || my < 0 || mx + w > mask_dev->w || my + h > mask_dev->h))) {
        set_error("sb_blender_feed_dev: invalid argument");
        return SB_ERR_INVALID;
    }
    if (!b->prepared) {
        set_error("sb_blender_feed_dev: prepare() has not been called");
        return SB_ERR_STATE;
    }
    const uint8_t *dimg = img->p + ((size_t)iy * img->w + ix) * 3;
    const uint8_t *dmask = mask_dev ? mask_dev->p + (size_t)my * mask_dev->w + mx : nullptr;
    return blender_feed_impl(b, nullptr, 0, 0, dimg, (size_t)img->w * 3, mask_host, mask_pitch, dmask, mask_dev ? (size_t)mask_dev->w : 0, w, h, tl_x,
                             tl_y);
}

int sb_blender_blend(sb_blender *b, uint8_t *dst, size_t dst_pitch, uint8_t *dst_mask, size_t mask_pitch, int16_t *dst_s16,
                     size_t s16_pitch)
{
    if (!b) {
        set_error("sb_blender_blend: null handle");
        return SB_ERR_INVALID;
    }
    if (!b->prepared) {
        set_error("sb_blender_blend: prepare() has not been called (or blend() was already called)");
        return SB_ERR_STATE;
    }
    const int w = b->plan.roi.w, h = b->plan.roi.h;
    if ((dst && dst_pitch < (size_t)w * 3) || (dst_mask && mask_pitch < (size_t)w) || (dst_s16 && s16_pitch < (size_t)w * 6)) {
        set_error("sb_blender_blend: destination pitch too small for roi width %d", w);
        return SB_ERR_INVALID;
    }
    SB_TRY(ensure_device());
    Staging st(default_stream());
    cudaStream_t s = st.stream();
    PanoOut out;
    std::memset(&out, 0, sizeof out);
    out.w = w;
    out.h = h;
    if (dst) {
        out.rgb = st.tmp<uint8_t>((size_t)w * 3 * h);
        out.rgb_pitch = (long long)w * 3;
    }
    if (dst_mask) {
        out.mask = st.tmp<uint8_t>((size_t)w * h);
        out.mask_pitch = w;
    }
    if (dst_s16) {
        out.s16 = st.tmp<int16_t>((size_t)w * 3 * h);
        out.s16_pitch = (long long)w * 3;
    }
    st.run([&] { return b->plan.allocate(s); });
    st.run([&] { return b->plan.run(out, s); });
    if (dst) st.down(dst, dst_pitch, out.rgb, (size_t)w * 3, (size_t)w * 3, h);
    if (dst_mask) st.down(dst_mask, mask_pitch, out.mask, w, w, h);
    if (dst_s16) st.down(dst_s16, s16_pitch, out.s16, (size_t)w * 6, (size_t)w * 6, h);
    const int rc = st.finish();
    // like OpenCV, blend() consumes the state, also when it fails: a new prepare() is needed before the next feed
    blender_drop_feeds(b);
    b->prepared = false;
    return rc;
}

}  // extern "C"
