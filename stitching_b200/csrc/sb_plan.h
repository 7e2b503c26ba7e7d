// sb_plan.h -- host-side plan of one blend: pano geometry, per-feed padded rects, pyramid storage in HBM.
#pragma once
#include <functional>
#include <string>
#include <utility>
#include <vector>

#include "sb_internal.h"

namespace sb {

struct Rect {
    int x, y, w, h;
};

// one recorded Blender.feed (level-0 data already resident in HBM)
struct FeedDesc {
    int w, h, tlx, tly;
    const uint32_t *rgbm;  // packed layout, or
    long long rgbm_pitch;
    const int16_t *s16;    // generic int16 layout (+ mask)
    long long s16_pitch;
    const uint8_t *mask;
    long long mask_pitch;
};

// derive blender.py:25-36's parameters: returns blend kind actually used and num_bands / sharpness
void derive_blend_params(int requested_kind, double blend_strength, const Rect &roi, int *kind, int *num_bands, float *sharpness);
Rect result_roi(const int *corners_xy, const int *sizes_wh, int n);  // cv.detail.resultRoi (blender.py:24)

class BlendPlan {
public:
    int kind = SB_BLEND_NO;
    int nb = 0;              // effective number of bands (after clipping)
    bool binary_masks = false;  // every fed mask byte is 0 or 255 (a compositor's validity masks): exact shortcut in pyrDown l0
    float sharpness = 0.f;
    Rect roi{0, 0, 0, 0};    // final (unpadded) pano roi
    int wp = 0, hp = 0;      // padded pano size (multiples of 2^nb)
    std::vector<FeedImage> imgs;  // host copy of the device descriptors
    PanoLevel pano[SB_MAX_BANDS + 1];
    FeedImage *imgs_dev = nullptr;
    PanoLevel *pano_dev = nullptr;
    ColDesc *col_dev = nullptr;  // [(nb+1)][n] compact descriptors for the fast kernels
    PyrDesc *pyr_dev = nullptr;
    std::vector<ColDesc> col_host;  // host copies (the sharded compositor builds its item lists from them)
    std::vector<PyrDesc> pyr_host;
    // tile kernels (sb_collapse_tile.cu): per-(level, image) descriptors; null when the plan does not qualify (generic
    // int16 feeds: the fast kernels then do the work) and in a sharded plan, whose strips get their own lists of images
    // and slabs (ShardPlan::tile_items_dev)
    TileDesc *tile_dev = nullptr;   // [(nb+1)][n]
    bool tile_images_ok = false;    // the images with storage on this device qualify for the tile kernels (sb_collapse_tile.cu)
    static TileDesc tile_desc(const FeedImage &im, int l);
    // fused pyramid tail (sb_tail.cu): levels >= tail_from run in one launch; tail_from > nb: no tail
    int tail_from = 1 << 30;
    unsigned *tail_state_dev = nullptr;  // the grid barrier's two words
    // images [active_first, active_first + active_count) get pyramid storage; the others (owned by other ranks of
    // a sharded composite) only take part in the geometry.  active_count < 0: all images.
    int active_first = 0, active_count = -1;

    // geometry only (no device work): usable without a GPU for tests of the host logic
    int set_geometry(int kind, int num_bands_requested, float sharpness, const Rect &roi);
    int add_feed(const FeedDesc &f);  // computes the padded rect; SB_ERR_INVALID if the feed leaves the roi
    // device storage for pyramid levels >= 1, feather weights, pano levels; uploads descriptors
    int allocate(cudaStream_t s);
    // enqueue all blend kernels; `mark` (optional) is called after each launch with its name (timing hooks)
    int run(const PanoOut &out, cudaStream_t s, const std::function<int(const std::string &)> &mark = nullptr);
    // multiband, pyrDown of level l -> l+1 for images [first, first + count)
    int pyrdown(int l, int first, int count, cudaStream_t s) const;
    // multiband, strip [x0, x1) of padded-pano columns (whole pano: [0, wp)): the columns [*a, *b) of level l it collapses,
    // and that collapse's arguments over n items `col` (`tile`: their tile descriptors, or null) into `out` (from column x0)
    void region_x(int x0, int x1, int l, int *a, int *b) const;
    CollapseArgs collapse_args(int l, int x0, int x1, const ColDesc *col, int n, const TileDesc *tile, const PanoOut &out) const;
    // compulsory HBM traffic per launch, in launch order: (name, bytes)
    std::vector<std::pair<std::string, double>> launch_bytes() const;
    void release(cudaStream_t s);
    double model_bytes(double *pyr, double *collapse) const;
    size_t arena_bytes() const { return arena_bytes_; }

private:
    void *arena_ = nullptr;
    size_t arena_bytes_ = 0;
};

}  // namespace sb
