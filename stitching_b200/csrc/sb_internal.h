// sb_internal.h -- shared declarations of libstitch_b200.so (not part of the public C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/stitch_b200.h"

#define SB_MAX_BANDS 16
#define SB_MAX_IMAGES 256
#define SB_SRC_PAD 16  // spare bytes after a source image: the warp kernel reads aligned 8-byte words
// cv::remap (under PyRotationWarper.warp) asserts every side of its source and result below SHRT_MAX: the warp entries and
// the compositor refuse sources and warped images with a side of this many pixels or more
#define SB_MAX_WARP_SIDE 32767

namespace sb {

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);
#define SB_CUDA(call)                                                         \
    do {                                                                      \
        cudaError_t e__ = (call);                                             \
        if (e__ != cudaSuccess) return sb::cuda_fail(e__, #call, __FILE__, __LINE__); \
    } while (0)
#define SB_TRY(call)            \
    do {                        \
        int r__ = (call);       \
        if (r__ != SB_OK) return r__; \
    } while (0)

int ensure_device();  // SB_OK when sb_init succeeded (or lazily selects device 0)
int sm_count();
void count_launch(unsigned n = 1);
void adjust_launch_count(long long delta);  // graph capture records launches that do not execute; replays execute them
cudaStream_t default_stream();

// page-locked host memory (cudaMallocHost), capped by SB_PINNED_MAX_BYTES when it is set (sb_context.cpp)
cudaError_t host_alloc_pinned(void **p, size_t bytes);
// stream-ordered device allocation (cudaMallocAsync pool with a high release threshold)
int dev_alloc(void **p, size_t bytes, cudaStream_t s);
void dev_free(void *p, cudaStream_t s);

// The device work of one call that reads or writes its caller's memory, on stream `s` (sb_context.cpp).  It keeps the
// temporaries, the buffers that outlive a successful call and the first failure; once a step has failed every later one is
// skipped (allocations return null).  finish() synchronises `s` on every path, so that no copy from or to the caller's
// memory is still in flight, and returns the first failure; the destructor does the same if finish() was not called, then
// frees the temporaries, and the kept buffers too when a step failed.
class Staging {
  public:
    explicit Staging(cudaStream_t s) : s_(s) {}
    ~Staging();
    Staging(const Staging &) = delete;
    Staging &operator=(const Staging &) = delete;
    cudaStream_t stream() const { return s_; }
    // a step that returns SB_OK or a failure whose message it has set
    template <typename F>
    void run(F &&step)
    {
        if (rc_ == SB_OK) rc_ = step();
    }
    template <typename T>
    T *tmp(size_t count) { return (T *)alloc(count * sizeof(T), tmps_); }
    template <typename T>
    T *keep(size_t count) { return (T *)alloc(count * sizeof(T), kept_); }
    const std::vector<void *> &kept() const { return kept_; }
    // `rows` rows of `width` bytes (row pitch `pitch`) between two buffers, as sb_copy2d
    void copy(void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t rows, cudaMemcpyKind kind);
    // a host rectangle into a new temporary of `rows` rows of `width` bytes
    template <typename T>
    T *up(const void *src, size_t pitch, size_t width, size_t rows)
    {
        T *d = (T *)alloc(width * rows, tmps_);
        copy(d, width, src, pitch, width, rows, cudaMemcpyHostToDevice);
        return d;
    }
    template <typename T>
    T *up(const std::vector<T> &v) { return up<T>(v.data(), v.size() * sizeof(T), v.size() * sizeof(T), 1); }
    void down(void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t rows)
    {
        copy(dst, dpitch, src, spitch, width, rows, cudaMemcpyDeviceToHost);
    }
    int finish();

  private:
    void *alloc(size_t bytes, std::vector<void *> &list);
    cudaStream_t s_;
    int rc_ = SB_OK;
    bool finished_ = false;
    std::vector<void *> tmps_, kept_;
};

// ---------------------------------------------------------------------------------------------
// geometry (host, libm): sb_geometry.cpp
// ---------------------------------------------------------------------------------------------
struct Projector {
    int type;  // SB_WARP_* (affine folded into plane; the A/B variants folded into their class, parameters in a, b)
    float scale;
    float a, b;  // compressedPlane / panini parameters
    float k[9], rinv[9], r_kinv[9], k_rinv[9], t[3];
};
void projector_setup(Projector &p, int warp_type, float scale, const float *K, const float *R);
void projector_roi(const Projector &p, int src_w, int src_h, int rect[4]);
// Separable backward-map tables: for output column u (absolute, tl.x + i) and row v
//   x_ = rowA[v] * colX[u];  y_ = rowY[v];  z_ = rowA[v] * colZ[u]
// (multiplication by an exact 1.0f keeps cylindrical / plane bit-identical to the unfactored form)
void projector_tables(const Projector &p, const int rect[4], float *colX, float *colZ, float *rowA, float *rowY);
// projections whose mapBackward is not separable: the float maps of RotationWarperBase::buildMaps over `rect`
// (rect[3] rows of rect[2] floats each), computed with libm on all host cores
bool projector_needs_maps(const Projector &p);
void projector_maps(const Projector &p, const int rect[4], float *xmap, float *ymap);

// ---------------------------------------------------------------------------------------------
// device-side descriptors
// ---------------------------------------------------------------------------------------------
struct WarpJob {
    const uint8_t *src;  // u8x3 interleaved
    int sw, sh;
    long long spitch;    // bytes
    const uint32_t *src4;  // optional: the same image as r | g<<8 | b<<16 (byte 3 zero), sw pixels per row (compositor: repacked at upload)
    uint8_t *dst_rgb;    // u8x3 interleaved or null
    long long dst_pitch;
    uint8_t *dst_mask;   // u8 or null
    long long mask_pitch;
    uint32_t *dst_rgbm;  // packed r | g<<8 | b<<16 | mask<<24, or null
    long long rgbm_pitch;  // elements
    int blend_mask_and;         // 1: the stored weight byte is blend_mask & validity (sb_compositor_set_seam_mask)
    const uint8_t *blend_mask;  // optional blend mask (seam mask AND validity, stitcher.py:223-239) stored in the
    long long blend_mask_pitch; // mask byte of dst_rgbm instead of the validity mask
    int dw, dh;
    const float *colX, *colZ, *rowA, *rowY;
    const float *xmap, *ymap;  // non-null: backward map given per pixel (dw floats per row), the tables are unused
    float k[9];
    int always_divide;  // plane / affine: x/z, y/z unconditionally
    float xin_hi, yin_hi;  // 32 (sw-1) - 0.5, 32 (sh-1) - 0.5: upper limits of x*32, y*32 for a footprint inside the image
    // exposure compensation of the warped image (ExposureErrorCompensator.apply, stitcher.py:219-221), fused into the
    // warp's epilogue.  gain_mode 0: none; 1: float32 gain map (gain_gc = 1 or 3 channels) resized to dw x dh through
    // the per-axis taps below (resize_f32_taps, TAPS_IPP); 2: scalar gains as three 256-entry tables
    // (gain_lut[c * 256 + value]); 3: as 1 for a map with a side of 1 (TAPS_COLS / TAPS_ROWS, OpenCV's own passes)
    int gain_mode, gain_gw, gain_gc, gain_pad;
    const float *gain_map;
    const int *gain_tx, *gain_ty;    // [i0 | i1], dw / dh entries each
    const float *gain_fx, *gain_fy;  // fractions
    const uint8_t *gain_lut;
};

// floats in the device tables of a w x h warp: colX, colZ (each padded to a multiple of 4), rowA, rowY
inline size_t warp_table_floats(int w, int h) { return (size_t)2 * ((w + 3) & ~3) + (size_t)2 * h; }

// one pyramid level of one fed image: planar int16 x3 + float32 weights
// Two colour layouts.  An image fed as bytes (RGBM) keeps every Gaussian level inside 0..255 (the 5x5 weights sum
// to 256), so its levels are stored as ONE WORD per pixel: q[y*pitch + x] = r | g << 8 | b << 16, byte 3 zero --
// the layout of level 0 without the mask byte.  The kernels split a word into two 16-bit lanes (r | b << 16 and g)
// after loading it, and red and blue run as the two lanes of one word through every filter (no lane ever carries:
// 256*255+128 < 2^16).
// A generic int16 feed (arbitrary values) keeps planar int16 and is served by the simple kernels only.
struct Level {
    uint32_t *q;       // [h][pitch] words, or null
    int16_t *g;        // [3][h][pitch] planar, or null
    float *w;          // [h][pitch]
    int w_px, h_px;    // level size
    int pitch;         // elements, for q / g rows and w rows
    long long plane;   // elements between colour planes of g
};

#define SB_DT_CHUNKS 32    // row chunks per column in the parallel column pass of the L1 distance transform
struct FeedImage {
    // level 0 (one of the two layouts)
    const uint32_t *rgbm;  // packed u8x3 + mask
    long long rgbm_pitch;  // elements
    const int16_t *s16;    // interleaved int16x3 (generic feed) or null
    long long s16_pitch;   // elements (int16)
    const uint8_t *mask;   // with s16 layout
    long long mask_pitch;
    int w, h;              // fed image size
    int left, top;         // image origin inside its padded rect
    int px, py;            // padded rect origin relative to the padded pano (level 0)
    int pw, ph;            // padded rect size (multiples of 2^nb)
    int dx, dy;            // feather / no: image origin relative to the pano roi
    const float *fw;       // feather weight map [h][w] (dense)
    int *dts;              // feather: scratch of the distance transform's column pass, [2][SB_DT_CHUNKS][w] ints
    Level lv[SB_MAX_BANDS + 1];  // lv[0] unused
};

// Compact per-(image, level) descriptors for the fast kernels: everything a kernel needs for one level in a
// few 16-byte words, prebuilt on the host (the generic FeedImage stays the source of truth for the simple ones).
struct alignas(16) ColDesc {       // collapse of level l
    int ox, oy, w_l, h_l;          // padded rect of the image at level l, pano level coordinates
    const uint32_t *rgbm;          // level 0: packed fed image
    union {
        const uint32_t *q;         // kind 0, level l >= 1: colour words
        const int16_t *g;          // kind 1: the slab's three int16 planes of partial sums
    };
    const float *w;                // weights (kind 1: weight sums)
    const uint32_t *uq;            // level l+1 colour words (null at the top level)
    int rgbm_pitch, iw, ih, left;  // level 0: image size and origin inside the padded rect
    int top, pitch, plane, upitch; // level l / l+1 pitches, in elements; plane: stride of a slab's planes
    int pad0, kind, pad1, pad2;    // kind 0: a fed image; 1: a slab of partial sums
};
struct alignas(16) PyrDesc {       // pyrDown of level l -> l+1
    int sw, sh, dpitch, pad3;      // source level size; destination pitch (elements)
    const uint32_t *rgbm;          // level 0 source
    const uint32_t *sq;            // level >= 1 source colour words
    const float *swt;
    uint32_t *dq;
    float *dwt;
    int rgbm_pitch, iw;
    int ih, left, top, spitch;
    int pad0, pad1, pad2, pad4;
};

// Per-(level, image) descriptor of the tile kernels (sb_collapse_tile.cu), next to the item's ColDesc: the rect that
// decides whether the item touches a tile (= the extent of its level-l source) and the origins of its staged windows.
struct alignas(16) TileDesc {
    int x0, y0, w, h;           // level 0: the fed IMAGE inside its padded rect (weights are 0 outside); levels >= 1: the padded rect
    int ox, oy, uw, uh;         // padded rect origin at this level; size of the next coarser level (source of the pyrUp)
};
// window shapes of the tile kernels (one CTA = TILE_W x TILE_H pixels of a level, one thread per two stacked 2x2 quads)
#define SB_TILE_W 64
#define SB_TILE_H 32
#define SB_TILE_UPW (SB_TILE_W / 2 + 2)   // 34: the 3x3 neighbourhoods of the tile's quads at the coarser level
#define SB_TILE_UPH (SB_TILE_H / 2 + 2)   // 18

struct PanoLevel {
    int16_t *c;  // collapsed planar int16 x3 [3][h][pitch]
    int w_px, h_px, pitch;
    long long plane;
};

struct PanoOut {
    uint8_t *rgb; long long rgb_pitch;     // final uint8 HxWx3 (nullable)
    uint8_t *mask; long long mask_pitch;   // final uint8 mask (nullable)
    int16_t *s16; long long s16_pitch;     // final int16 HxWx3 before convertScaleAbs (nullable); pitch in elements
    int w, h;                              // unpadded roi size
};

// one launch of the fast per-level multiband kernel (sb_collapse_fast.cu), passed by value
#define SB_MAX_ITEMS 320  // fed images + slabs of other ranks
struct CollapseArgs {
    const ColDesc *col;       // items of this level in feed order (device)
    int n;
    PanoLevel up, cur;        // C_{l+1} (source of the pyrUp) and C_l (destination)
    int rx0, ry0, rw, rh;     // region of the level covered by this launch (even-aligned below the top level)
    int partial;              // 1: write the partial sums (acc, wsum) of the items to the slab below instead of finishing
    int16_t *slab_acc;        //    int16 x3 planes, origin = (rx0, ry0)
    float *slab_w;
    int slab_pitch, slab_plane;
    PanoOut out;              // level 0: final outputs; the buffer covers pano columns [out_x0, out_x0 + out.w)
    int out_x0, out_lo, out_hi;  // only columns [out_lo, out_hi) are stored (a strip's margin is not output)
    const TileDesc *tile;     // tile kernels: items of this level, same order as col (null: not available for this launch)
    int has_slabs;            // some items are slabs of partial sums (ColDesc kind 1): the tile kernels' slab instantiation
};
// the per-level multiband kernel over A's region: the shared-memory tile kernel where A.tile is given and the launch
// qualifies, else k_collapse_fast (sb_collapse_fast.cu)
int launch_collapse(const CollapseArgs &A, int l, int nb, cudaStream_t s);
// the tile kernel alone (sb_collapse_tile.cu); returns SB_ERR_STATE when the launch does not qualify
int launch_collapse_tile(const CollapseArgs &A, int l, int nb, cudaStream_t s);
bool collapse_tile_enabled();

// ---------------------------------------------------------------------------------------------
// kernel launchers
// ---------------------------------------------------------------------------------------------
// jobs are HOST structs: they are passed by value in the kernel parameter block, SB_WARP_BATCH images per launch
#define SB_WARP_BATCH 32
int launch_warp(const WarpJob *jobs_host, int n_jobs, cudaStream_t s);
// the device tables (`tab_dev`, warp_table_floats(w, h)) and the job of one image warped to `rect`; the upload reads
// `host_tab` until `s` is synchronised (sb_jobs.cpp)
int make_warp_job(const Projector &p, const int rect[4], int src_w, int src_h, float *tab_dev, WarpJob *job, cudaStream_t s,
                  std::vector<float> &host_tab);
int warp_maps_upload(const Projector &p, const int rect[4], float *maps_dev, WarpJob *job, cudaStream_t s);  // sb_jobs.cpp
// u8x3 contiguous (w * h pixels) -> r | g<<8 | b<<16 words (the compositor's source layout for the warp kernel)
int launch_repack_rgbx(const uint8_t *rgb, uint32_t *dst, long long pixels, cudaStream_t s);
// launch_warp's kernel choice for a batch of jobs: true when it reads WarpJob::src4 of jobs that have one (sb_warp.cu)
bool warp_batch_rgbm(const WarpJob *jobs, int cnt);
// one image of k_resize_src: Images.resize_img_by_scaler (cv.resize INTER_LINEAR_EXACT) from a camera-size frame into
// the warp's source layout, in place of the repack (sb_compositor_opts.in_w / in_h)
struct ResizeJob {
    const uint8_t *src;  // camera-size u8x3, rows of 3 * sw bytes, SB_SRC_PAD spare bytes after the last
    uint32_t *dst4;      // FINAL size, one word per pixel (WarpJob::src4), or null:
    uint8_t *dst3;       //   then FINAL size, packed u8x3 (WarpJob::src)
    const int *tx, *ty;  // device taps [i0 | i1 | c1] of the two axes (resize_exact_taps), dw / dh entries each
    int sw, dw;
    long long px;        // dw * dh
};
struct ResizeBatch {
    ResizeJob j[SB_WARP_BATCH];
};
int launch_resize_src(const ResizeJob *jobs, int n_jobs, cudaStream_t s);  // one launch per SB_WARP_BATCH images
int launch_pack_rgbm(const uint8_t *rgb, long long rgb_pitch, const uint8_t *mask, long long mask_pitch, uint32_t *dst,
                     long long dst_pitch, int w, int h, cudaStream_t s);
// level `l` -> `l+1` of images [first, first+count)
// `pyr`: the compact descriptors of level l of all images (device pointer, indexed like imgs_host)
// binary_masks: the caller guarantees that every mask byte of these images is 0 or 255 (used for l <= 2; sb_pyrdown_fast.cu)
int launch_pyrdown(const FeedImage *imgs_dev, const FeedImage *imgs_host, const PyrDesc *pyr, int first, int count, int l,
                   cudaStream_t s, bool binary_masks);
// SB_KERNELS=simple selects the one-thread-per-pixel gather kernels everywhere (debugging / A-B parity)
bool use_simple_kernels();
// multiband with the gather kernel (generic int16 feeds, SB_KERNELS=simple, no bands): accumulate + normalise + collapse
// level l (top-down) of the lw x lh level; at l == 0 writes the final outputs
int launch_collapse_gather(const FeedImage *imgs_dev, int n, const PanoLevel *pano_dev, int l, int nb, int lw, int lh, PanoOut out,
                           cudaStream_t s);
// feather: distance-transform weight maps, then one fused accumulate/normalise pass; NO blender
// levels T .. nb in one launch (sb_tail.cu); SB_ERR_STATE: not available (emulation build), launch per level instead
int launch_tail(const FeedImage *imgs_dev, const PanoLevel *pano_dev, int first, int count, int n, int T, int nb, int wp, int hp, const PanoOut &out,
                unsigned *state, cudaStream_t s);
int launch_feather_weights(const FeedImage *imgs_dev, const FeedImage *imgs_host, int n, float sharpness, cudaStream_t s);
int launch_simple_blend(const FeedImage *imgs_dev, int n, int feather, PanoOut out, cudaStream_t s);
// sharded feather blend: a slab of partial sums (acc int16 x3 planes with wrap-around, wsum float32) over a rectangle of
// the pano roi, and one launch over a region: the slabs of lower ranks, images [i0, i1), the slabs of higher ranks, in that
// order; `partial`: write the sums as a slab instead of normalising
struct FeatherSlab {
    int x0, y0, w, h, pitch, plane;
    const int16_t *acc;
    const float *wsum;
};
struct FeatherRegionArgs {
    const FeedImage *imgs;
    int i0, i1;
    const FeatherSlab *slabs;
    int n_before, n_after;
    int rx0, ry0, rw, rh;    // region, pano-roi coordinates
    int partial;
    int16_t *slab_acc;       // partial: origin = (rx0, ry0)
    float *slab_w;
    int slab_pitch, slab_plane;
    PanoOut out;             // !partial: the buffer's origin is pano pixel (out_x0, out_y0)
    int out_x0, out_y0;
};
int launch_feather_region(const FeatherRegionArgs &A, cudaStream_t s);
int launch_flush_l2(void *buf, size_t bytes, cudaStream_t s);
int launch_wait_flags(const unsigned *flags, unsigned mask, unsigned value, cudaStream_t s);  // lanes with a mask bit wait for flags[lane] >= value
// ExposureErrorCompensator.apply: taps of the float32 bilinear resize of a gain map (sb_geometry.cpp), the 256-entry
// table of a scalar gain, and the host-buffer entry's kernel (sb_warp.cu)
enum { TAPS_IPP = 0, TAPS_COLS = 1, TAPS_ROWS = 2 };  // resize_f32_taps' forms
void resize_f32_taps(int n_src, int n_dst, int *i0i1, float *fr, int form);  // i0i1: 2 * n_dst ints
void gain_scalar_lut(const double gain[3], uint8_t lut[768]);
// rows copy; a fully contiguous image goes as ONE linear transfer (the DMA engines reach PCIe line rate with those)
static inline cudaError_t sb_copy2d(void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t height,
                                    cudaMemcpyKind kind, cudaStream_t s)
{
    if (dpitch == width && spitch == width) return cudaMemcpyAsync(dst, src, width * height, kind, s);
    return cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, kind, s);
}

// Timelapser frame: src8 (uint8 x3, pitch in bytes) or src16 (int16 x3, pitch in ELEMENTS) pasted at (dx, dy) of a cw x ch canvas
int launch_timelapse_frame(const uint8_t *src8, const int16_t *src16, long long spitch, int sw, int sh, int dx, int dy, uint8_t *dst,
                           long long dpitch, int cw, int ch, cudaStream_t s);
// one image of k_timelapse_paste: the warped part of a timelapse frame (rgbm, w x h words) as dense u8x3 rows of w * 3
// bytes at dst (16-byte aligned)
struct PasteJob {
    const uint32_t *rgbm;
    uint8_t *dst;
    long long rgbm_pitch;  // elements
    int w, h;
};
int launch_timelapse_paste(const PasteJob *jobs_dev, int n_jobs, long long max_bytes, cudaStream_t s);  // one launch for all
int launch_gain_apply(uint8_t *img, long long pitch, int w, int h, const WarpJob &gain_fields, cudaStream_t s);
// device copies of one image's gain (map + taps for a w x h target, or the scalar tables) and the WarpJob fields for them
struct GainData {
    float *map = nullptr, *fx = nullptr, *fy = nullptr;
    int *tx = nullptr, *ty = nullptr;
    uint8_t *lut = nullptr;
};
// sub (nullable): only the rect sub = (x, y, w', h') of the w x h image is warped; the map is still resized to w x h and the
// job indexes the taps of that rect's columns and rows
int gain_upload(WarpJob *job, GainData *gd, int w, int h, const float *gain_map, int gw, int gh, int gc, const double *gain_scalar,
                cudaStream_t s, const int *sub = nullptr);  // synchronises s
void gain_free(GainData *gd, cudaStream_t s);
// Images.resize_img_by_scaler: cv.resize(uint8, INTER_LINEAR_EXACT) (sb_seam.cu, sb_geometry.cpp)
void resize_exact_taps(int n_src, int n_dst, int *t);  // t: 3 * n_dst ints
int launch_resize_exact(const uint8_t *src, long long spitch, int cn, const int *tx, const int *ty, uint8_t *dst, long long dpitch, int w,
                        int h, cudaStream_t s);
// SeamFinder.resize (sb_seam.cu, sb_geometry.cpp)
void resize_linear_taps(int n_src, int n_dst, bool columns, int *t);  // t: 4 * n_dst ints
int launch_seam_resize(const uint8_t *seam, int sw, int sh, uint8_t *scratch, const int *tx, const int *ty, const uint8_t *mask,
                       long long mask_pitch, uint8_t *dst, long long dst_pitch, int w, int h, cudaStream_t s);
// device version of SeamFinder.resize for host or device `mask` / `dst` buffers already on the device: uploads the seam
// mask, builds the taps, runs the two kernels (synchronises `s`)
int seam_resize_device(const uint8_t *seam_host, size_t seam_pitch, int sw, int sh, const uint8_t *mask_dev, long long mask_pitch,
                       uint8_t *dst_dev, long long dst_pitch, int w, int h, cudaStream_t s);
int launch_selftest_division(unsigned long long n, unsigned long long seed, int mode, unsigned long long *bad_dev, cudaStream_t s);

}  // namespace sb
