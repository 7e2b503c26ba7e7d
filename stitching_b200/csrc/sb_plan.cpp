// sb_plan.cpp -- geometry and storage plan of one blend (host logic; no kernels in this file).
//
// Restates the bookkeeping of stitching/blender.py:23-38 (Blender.prepare: resultRoi, blend width,
// num_bands / sharpness) and of MultiBandBlender::prepare / ::feed's rect arithmetic (SURVEY.md A.4
// steps 0-1): band clipping, padding the pano to a multiple of 2^nb, the per-feed padded rect.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "sb_plan.h"

namespace sb {

namespace {
inline int round_up(int v, int a) { return v + (a - v % a) % a; }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline int level_pitch(int w) { return (int)align_up((size_t)std::max(w, 1), 64); }  // elements: 128 B of int16
}  // namespace

Rect result_roi(const int *corners_xy, const int *sizes_wh, int n)
{
    int x0 = corners_xy[0], y0 = corners_xy[1], x1 = x0 + sizes_wh[0], y1 = y0 + sizes_wh[1];
    for (int i = 1; i < n; ++i) {
        x0 = std::min(x0, corners_xy[2 * i]);
        y0 = std::min(y0, corners_xy[2 * i + 1]);
        x1 = std::max(x1, corners_xy[2 * i] + sizes_wh[2 * i]);
        y1 = std::max(y1, corners_xy[2 * i + 1] + sizes_wh[2 * i + 1]);
    }
    return Rect{x0, y0, x1 - x0, y1 - y0};
}

void derive_blend_params(int requested_kind, double blend_strength, const Rect &roi, int *kind, int *num_bands, float *sharpness)
{
    // blender.py:25  blend_width = sqrt(w*h) * strength / 100 (double)
    const double blend_width = std::sqrt((double)roi.w * (double)roi.h) * blend_strength / 100.0;
    *num_bands = 0;
    *sharpness = 0.f;
    if (requested_kind == SB_BLEND_NO || blend_width < 1.0) {
        *kind = SB_BLEND_NO;  // blender.py:27-28
    } else if (requested_kind == SB_BLEND_MULTIBAND) {
        *kind = SB_BLEND_MULTIBAND;
        *num_bands = (int)(std::log(blend_width) / std::log(2.0) - 1.0);  // blender.py:32, truncation
    } else {
        *kind = SB_BLEND_FEATHER;
        *sharpness = (float)(1.0 / blend_width);  // blender.py:36
    }
}

int BlendPlan::set_geometry(int kind_, int num_bands_requested, float sharpness_, const Rect &roi_)
{
    if (roi_.w <= 0 || roi_.h <= 0) {
        set_error("prepare: empty roi %dx%d", roi_.w, roi_.h);
        return SB_ERR_INVALID;
    }
    kind = kind_;
    sharpness = sharpness_;
    roi = roi_;
    imgs.clear();
    nb = 0;
    wp = roi.w;
    hp = roi.h;
    if (kind == SB_BLEND_MULTIBAND) {
        if (num_bands_requested < 0) {
            set_error("prepare: negative number of bands %d", num_bands_requested);
            return SB_ERR_INVALID;
        }
        // MultiBandBlender::prepare: crop unnecessary bands, then pad the pano so every level halves exactly
        const double max_len = (double)std::max(roi.w, roi.h);
        const int limit = (int)std::ceil(std::log(max_len) / std::log(2.0));
        nb = std::min(num_bands_requested, limit);
        if (nb > SB_MAX_BANDS) {
            set_error("prepare: %d bands exceed SB_MAX_BANDS=%d", nb, SB_MAX_BANDS);
            return SB_ERR_INVALID;
        }
        wp = round_up(roi.w, 1 << nb);
        hp = round_up(roi.h, 1 << nb);
    }
    return SB_OK;
}

int BlendPlan::add_feed(const FeedDesc &f)
{
    if (f.w <= 0 || f.h <= 0) {
        set_error("feed: empty image %dx%d", f.w, f.h);
        return SB_ERR_INVALID;
    }
    if ((int)imgs.size() >= SB_MAX_IMAGES) {
        set_error("feed: more than %d images", SB_MAX_IMAGES);
        return SB_ERR_INVALID;
    }
    FeedImage im;
    std::memset(&im, 0, sizeof im);
    im.rgbm = f.rgbm;
    im.rgbm_pitch = f.rgbm_pitch;
    im.s16 = f.s16;
    im.s16_pitch = f.s16_pitch;
    im.mask = f.mask;
    im.mask_pitch = f.mask_pitch;
    im.w = f.w;
    im.h = f.h;
    im.dx = f.tlx - roi.x;
    im.dy = f.tly - roi.y;
    if (kind != SB_BLEND_MULTIBAND) {
        if (im.dx < 0 || im.dy < 0 || im.dx + f.w > roi.w || im.dy + f.h > roi.h) {
            set_error("feed: image rect (%d,%d %dx%d) leaves the prepared roi (%d,%d %dx%d)", f.tlx, f.tly, f.w, f.h, roi.x, roi.y, roi.w, roi.h);
            return SB_ERR_INVALID;
        }
        imgs.push_back(im);
        return SB_OK;
    }
    // MultiBandBlender::feed: keep the image with a gap of 3*2^nb around it, clipped to the padded pano;
    // snap the origin down and the extent up to the 2^nb lattice anchored at the pano origin.
    const int a = 1 << nb, gap = 3 * a;
    const int rx1 = roi.x + wp, ry1 = roi.y + hp;
    int x0 = std::max(roi.x, f.tlx - gap), y0 = std::max(roi.y, f.tly - gap);
    int x1 = std::min(rx1, f.tlx + f.w + gap), y1 = std::min(ry1, f.tly + f.h + gap);
    x0 = roi.x + (((x0 - roi.x) >> nb) << nb);
    y0 = roi.y + (((y0 - roi.y) >> nb) << nb);
    int ww = x1 - x0, hh = y1 - y0;
    if (ww <= 0 || hh <= 0) {
        set_error("feed: image rect (%d,%d %dx%d) does not intersect the prepared roi", f.tlx, f.tly, f.w, f.h);
        return SB_ERR_INVALID;
    }
    ww = round_up(ww, a);
    hh = round_up(hh, a);
    // shift back inside the padded pano if the rounded rect sticks out (never triggers: the lattice is
    // anchored at the pano origin and the padded pano size is a lattice multiple; kept for fidelity)
    const int sx = std::max(x0 + ww - rx1, 0), sy = std::max(y0 + hh - ry1, 0);
    x0 -= sx;
    y0 -= sy;
    im.left = f.tlx - x0;
    im.top = f.tly - y0;
    const int right = x0 + ww - f.tlx - f.w, bottom = y0 + hh - f.tly - f.h;
    if (im.left < 0 || im.top < 0 || right < 0 || bottom < 0) {
        set_error("feed: image rect (%d,%d %dx%d) leaves the prepared roi (%d,%d %dx%d)", f.tlx, f.tly, f.w, f.h, roi.x, roi.y, roi.w, roi.h);
        return SB_ERR_INVALID;
    }
    im.px = x0 - roi.x;
    im.py = y0 - roi.y;
    im.pw = ww;
    im.ph = hh;
    imgs.push_back(im);
    return SB_OK;
}

TileDesc BlendPlan::tile_desc(const FeedImage &im, int l)
{
    TileDesc t;
    std::memset(&t, 0, sizeof t);
    t.ox = im.px >> l;
    t.oy = im.py >> l;
    if (l == 0) {
        t.x0 = im.px + im.left;
        t.y0 = im.py + im.top;
        t.w = im.w;
        t.h = im.h;
    } else {
        t.x0 = t.ox;
        t.y0 = t.oy;
        t.w = im.pw >> l;
        t.h = im.ph >> l;
    }
    t.uw = im.pw >> (l + 1);
    t.uh = im.ph >> (l + 1);
    return t;
}

int BlendPlan::allocate(cudaStream_t s)
{
    release(s);
    const int n = (int)imgs.size();
    // carve every buffer out of one arena
    size_t off = 0;
    auto carve = [&](size_t bytes) {
        size_t o = off;
        off = align_up(off + bytes, 256);
        return o;
    };
    struct Slot { size_t g, w; };
    std::vector<std::vector<Slot>> slots(n);
    std::vector<size_t> fw_off(n, 0), dts_off(n, 0);
    size_t pano_off[SB_MAX_BANDS + 1] = {0};
    auto active = [&](int i) { return active_count < 0 || (i >= active_first && i < active_first + active_count); };
    if (kind == SB_BLEND_MULTIBAND) {
        for (int i = 0; i < n; ++i) {
            slots[i].resize(nb + 1);
            if (!active(i)) continue;  // another rank owns this image: geometry only
            for (int l = 1; l <= nb; ++l) {
                const int w = imgs[i].pw >> l, h = imgs[i].ph >> l, pitch = level_pitch(w);
                // byte-fed images: one word per pixel; generic int16 feeds: three int16 planes
                slots[i][l].g = carve(imgs[i].rgbm ? (size_t)h * pitch * sizeof(uint32_t) : (size_t)3 * h * pitch * sizeof(int16_t));
                slots[i][l].w = carve((size_t)h * pitch * sizeof(float));
            }
        }
        for (int l = 1; l <= nb; ++l) {
            const int w = wp >> l, h = hp >> l, pitch = level_pitch(w);
            pano_off[l] = carve((size_t)3 * h * pitch * sizeof(int16_t));
        }
    } else if (kind == SB_BLEND_FEATHER) {
        for (int i = 0; i < n; ++i)
            if (active(i)) {
                fw_off[i] = carve((size_t)imgs[i].w * imgs[i].h * sizeof(float));
                dts_off[i] = carve((size_t)2 * SB_DT_CHUNKS * imgs[i].w * sizeof(int));
            }
    }
    const size_t imgs_off = carve(sizeof(FeedImage) * (size_t)std::max(n, 1));
    const size_t panod_off = carve(sizeof(PanoLevel) * (SB_MAX_BANDS + 1));
    const size_t col_off = carve(sizeof(ColDesc) * (size_t)std::max(n, 1) * (nb + 1));
    const size_t pyr_off = carve(sizeof(PyrDesc) * (size_t)std::max(n, 1) * (nb + 1));
    const size_t tile_off = carve(sizeof(TileDesc) * (size_t)std::max(n, 1) * (nb + 1));
    const size_t tail_off = carve(256);
    arena_bytes_ = off;
    SB_TRY(dev_alloc(&arena_, arena_bytes_, s));
    // zero once: the row padding of every level (pitch - width elements, never written by a kernel) is read as part of
    // 16-byte chunks by the tile kernels' staged copies and must be "weight 0"
    SB_CUDA(cudaMemsetAsync(arena_, 0, arena_bytes_, s));
    char *base = (char *)arena_;
    std::memset(pano, 0, sizeof pano);
    if (kind == SB_BLEND_MULTIBAND) {
        for (int i = 0; i < n; ++i)
            for (int l = 1; l <= nb; ++l) {
                Level &L = imgs[i].lv[l];
                L.w_px = imgs[i].pw >> l;
                L.h_px = imgs[i].ph >> l;
                L.pitch = level_pitch(L.w_px);
                L.plane = (long long)L.h_px * L.pitch;
                L.q = active(i) && imgs[i].rgbm ? (uint32_t *)(base + slots[i][l].g) : nullptr;
                L.g = active(i) && !imgs[i].rgbm ? (int16_t *)(base + slots[i][l].g) : nullptr;
                L.w = active(i) ? (float *)(base + slots[i][l].w) : nullptr;
            }
        for (int l = 1; l <= nb; ++l) {
            PanoLevel &P = pano[l];
            P.w_px = wp >> l;
            P.h_px = hp >> l;
            P.pitch = level_pitch(P.w_px);
            P.plane = (long long)P.h_px * P.pitch;
            P.c = (int16_t *)(base + pano_off[l]);
        }
    } else if (kind == SB_BLEND_FEATHER) {
        for (int i = 0; i < n; ++i) {
            imgs[i].fw = active(i) ? (const float *)(base + fw_off[i]) : nullptr;
            imgs[i].dts = active(i) ? (int *)(base + dts_off[i]) : nullptr;
        }
    }
    imgs_dev = (FeedImage *)(base + imgs_off);
    pano_dev = (PanoLevel *)(base + panod_off);
    col_dev = (ColDesc *)(base + col_off);
    pyr_dev = (PyrDesc *)(base + pyr_off);
    tail_state_dev = (unsigned *)(base + tail_off);
    // fused tail (sb_tail.cu): OFF by default -- where it was measured, the one-launch per-pixel version of levels
    // 3..7 was slower than the twelve tuned per-level launches.
    // SB_TAIL_FROM=<level> enables it from that level on (A/B measurements, tests).
    tail_from = 1 << 30;
    if (kind == SB_BLEND_MULTIBAND && active_count < 0 && n > 0) {
        static const int forced = [] {
            const char *e = getenv("SB_TAIL_FROM");
            return e ? atoi(e) : -1;
        }();
        if (forced >= 0 && forced < nb) tail_from = forced;
    }
    // compact per-(level, image) descriptors for the fast kernels: [l * n + i]
    std::vector<ColDesc> &col = col_host;
    std::vector<PyrDesc> &pyr = pyr_host;
    col.assign((size_t)n * (nb + 1), ColDesc{});
    pyr.assign((size_t)n * (nb + 1), PyrDesc{});
    if (kind == SB_BLEND_MULTIBAND) {
        for (int l = 0; l <= nb; ++l)
            for (int i = 0; i < n; ++i) {
                const FeedImage &im = imgs[i];
                ColDesc &c = col[(size_t)l * n + i];
                std::memset(&c, 0, sizeof c);
                c.ox = im.px >> l;
                c.oy = im.py >> l;
                c.w_l = im.pw >> l;
                c.h_l = im.ph >> l;
                c.rgbm = im.rgbm;
                c.rgbm_pitch = (int)im.rgbm_pitch;
                c.iw = im.w;
                c.ih = im.h;
                c.left = im.left;
                c.top = im.top;
                if (l >= 1) {
                    c.q = im.lv[l].q;
                    c.w = im.lv[l].w;
                    c.pitch = im.lv[l].pitch;
                }
                if (l < nb) {
                    c.uq = im.lv[l + 1].q;
                    c.upitch = im.lv[l + 1].pitch;
                }
                PyrDesc &p = pyr[(size_t)l * n + i];
                std::memset(&p, 0, sizeof p);
                if (l < nb) {
                    p.sw = im.pw >> l;
                    p.sh = im.ph >> l;
                    p.rgbm = im.rgbm;
                    p.rgbm_pitch = (int)im.rgbm_pitch;
                    p.iw = im.w;
                    p.ih = im.h;
                    p.left = im.left;
                    p.top = im.top;
                    if (l >= 1) {
                        p.sq = im.lv[l].q;
                        p.swt = im.lv[l].w;
                        p.spitch = im.lv[l].pitch;
                    }
                    p.dq = im.lv[l + 1].q;
                    p.dwt = im.lv[l + 1].w;
                    p.dpitch = im.lv[l + 1].pitch;
                }
            }
        if (n) {
            SB_CUDA(cudaMemcpyAsync(col_dev, col.data(), sizeof(ColDesc) * col.size(), cudaMemcpyHostToDevice, s));
            SB_CUDA(cudaMemcpyAsync(pyr_dev, pyr.data(), sizeof(PyrDesc) * pyr.size(), cudaMemcpyHostToDevice, s));
        }
        // tile kernels (sb_collapse_tile.cu): per-(level, image) rects.  Byte-fed images with storage on this device;
        // the staged copies need 16-byte rows (RGBM pitch a multiple of 4 pixels, 16-byte aligned base)
        tile_dev = nullptr;
        tile_images_ok = n > 0 && nb >= 1 && collapse_tile_enabled();
        for (int i = 0; i < n && tile_images_ok; ++i)
            if (active(i)) tile_images_ok = imgs[i].rgbm != nullptr && imgs[i].rgbm_pitch % 4 == 0 && ((uintptr_t)imgs[i].rgbm & 15) == 0;
        const bool tiles = tile_images_ok && active_count < 0;  // (a sharded plan builds its own item lists: ShardPlan::allocate)
        if (tiles) {
            std::vector<TileDesc> td((size_t)n * (nb + 1));
            for (int l = 0; l <= nb; ++l)
                for (int i = 0; i < n; ++i) td[(size_t)l * n + i] = tile_desc(imgs[i], l);
            tile_dev = (TileDesc *)(base + tile_off);
            SB_CUDA(cudaMemcpyAsync(tile_dev, td.data(), sizeof(TileDesc) * td.size(), cudaMemcpyHostToDevice, s));
            SB_CUDA(cudaStreamSynchronize(s));  // `td` is a local
        }
    }
    if (n) SB_CUDA(cudaMemcpyAsync(imgs_dev, imgs.data(), sizeof(FeedImage) * n, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(pano_dev, pano, sizeof pano, cudaMemcpyHostToDevice, s));
    // the descriptor copies read pageable host memory owned by this object: make them complete now
    SB_CUDA(cudaStreamSynchronize(s));
    return SB_OK;
}

void BlendPlan::release(cudaStream_t s)
{
    if (arena_) dev_free(arena_, s);
    arena_ = nullptr;
    arena_bytes_ = 0;
    imgs_dev = nullptr;
    pano_dev = nullptr;
    col_dev = nullptr;
    pyr_dev = nullptr;
    tile_dev = nullptr;
    tail_state_dev = nullptr;
}

int BlendPlan::pyrdown(int l, int first, int count, cudaStream_t s) const
{
    return launch_pyrdown(imgs_dev, imgs.data(), pyr_dev + (size_t)l * imgs.size(), first, count, l, s, binary_masks);
}

void BlendPlan::region_x(int x0, int x1, int l, int *a, int *b) const
{
    *a = std::max(0, (x0 >> l) - 2);  // the margin the pyrUp of the next finer level reads
    *b = std::min(wp >> l, (x1 >> l) + 2);
    if (l == 0) {  // nothing finer reads level 0: no margin, and nothing beyond the (even-rounded) roi
        *a = x0;
        *b = std::min(x1, (roi.w + 1) / 2 * 2);
    }
    if (*b < *a) *b = *a;
}

CollapseArgs BlendPlan::collapse_args(int l, int x0, int x1, const ColDesc *col, int n, const TileDesc *tile, const PanoOut &out) const
{
    CollapseArgs A;
    std::memset(&A, 0, sizeof A);
    A.col = col;
    A.n = n;
    if (l < nb) A.up = pano[l + 1];
    A.cur = pano[l];
    int b;
    region_x(x0, x1, l, &A.rx0, &b);
    A.rw = b - A.rx0;
    A.rh = l == 0 ? (roi.h + 1) / 2 * 2 : hp >> l;
    A.out = out;
    A.out_x0 = x0;
    A.out_lo = std::min(x0, roi.w);  // the strip's own columns of the roi
    A.out_hi = std::min(x1, roi.w);
    A.tile = tile;
    return A;
}

int BlendPlan::run(const PanoOut &out, cudaStream_t s, const std::function<int(const std::string &)> &mark)
{
    const int n = (int)imgs.size();
    auto note = [&](const std::string &name) -> int { return mark ? mark(name) : SB_OK; };
    if (kind == SB_BLEND_MULTIBAND) {
        // the fast collapse needs byte-fed images (RGBM level 0, one colour word per pixel above) and at least one band
        bool fast = !use_simple_kernels() && nb >= 1;
        for (const FeedImage &im : imgs) fast = fast && im.rgbm != nullptr;
        int T = tail_from <= nb ? tail_from : nb + 1;  // levels >= T: one launch (sb_tail.cu)
        bool tail_done = false;
        for (int l = 0; l < nb; ++l) {
            if (l >= T) {
                if (tail_done) continue;
                const int rc = launch_tail(imgs_dev, pano_dev, 0, n, n, T, nb, wp, hp, out, tail_state_dev, s);
                if (rc == SB_OK) {
                    tail_done = true;
                    SB_TRY(note("tail_l" + std::to_string(T) + "-" + std::to_string(nb)));
                    continue;
                }
                if (rc != SB_ERR_STATE) return rc;
                T = nb + 1;  // not available here: per-level launches
            }
            SB_TRY(pyrdown(l, 0, n, s));
            SB_TRY(note("pyrdown_l" + std::to_string(l)));
        }
        for (int l = nb; l >= 0; --l) {
            if (tail_done && l >= T) continue;
            if (fast)
                SB_TRY(launch_collapse(collapse_args(l, 0, wp, col_dev + (size_t)l * n, n, tile_dev ? tile_dev + (size_t)l * n : nullptr, out),
                                       l, nb, s));
            else
                SB_TRY(launch_collapse_gather(imgs_dev, n, pano_dev, l, nb, wp >> l, hp >> l, out, s));
            SB_TRY(note("collapse_l" + std::to_string(l)));
        }
    } else {
        if (kind == SB_BLEND_FEATHER) {
            SB_TRY(launch_feather_weights(imgs_dev, imgs.data(), n, sharpness, s));
            SB_TRY(note("feather_weights"));
        }
        SB_TRY(launch_simple_blend(imgs_dev, n, kind == SB_BLEND_FEATHER, out, s));
        SB_TRY(note(kind == SB_BLEND_FEATHER ? "feather_blend" : "no_blend"));
    }
    return SB_OK;
}

// Compulsory HBM traffic of this plan's kernels in the layouts the levels are stored in (every input byte read once,
// every output byte written once, no accumulator round trips): see DESIGN.md "byte model".  Same order as run()'s launches.
std::vector<std::pair<std::string, double>> BlendPlan::launch_bytes() const
{
    std::vector<std::pair<std::string, double>> v;
    const double l0 = imgs.empty() ? 4.0 : (imgs[0].rgbm ? 4.0 : 7.0);  // bytes per level-0 pixel
    if (kind == SB_BLEND_MULTIBAND) {
#ifdef SB_EMU
        const int T = nb + 1;
#else
        const int T = tail_from <= nb ? tail_from : nb + 1;
#endif
        // bytes per pixel of a level >= 1 (colours + weight) and of its colours alone: one word + a float for byte-fed
        // images, three int16 + a float for generic int16 feeds
        auto lv_px = [](const FeedImage &im) { return im.rgbm ? 4.0 + 4.0 : 6.0 + 4.0; };
        auto rgb_px = [](const FeedImage &im) { return im.rgbm ? 4.0 : 6.0; };
        double tail = 0;
        for (int l = 0; l < nb; ++l) {
            double b = 0;
            for (const FeedImage &im : imgs) {
                const double src = (double)(im.pw >> l) * (im.ph >> l);
                b += (l == 0 ? l0 : lv_px(im)) * src + lv_px(im) * src / 4;  // read level l, write level l+1
            }
            if (l >= T)
                tail += b;
            else
                v.emplace_back("pyrdown_l" + std::to_string(l), b);
        }
        for (int l = nb; l >= 0; --l) {
            double b = 0;
            for (const FeedImage &im : imgs) {
                const double a = (double)(im.pw >> l) * (im.ph >> l);
                b += (l == 0 ? l0 : lv_px(im)) * a;   // G_l, W_l
                if (l < nb) b += rgb_px(im) * a / 4;  // G_{l+1} for the pyrUp
            }
            const double P = (double)(wp >> l) * (hp >> l);
            if (l < nb) b += 6.0 * P / 4;        // C_{l+1}
            b += l > 0 ? 6.0 * P : 4.0 * (double)roi.w * roi.h;  // C_l, or the final uint8x3 + mask
            if (l >= T) {
                tail += b;
                if (l == T) v.emplace_back("tail_l" + std::to_string(T) + "-" + std::to_string(nb), tail);
            } else {
                v.emplace_back("collapse_l" + std::to_string(l), b);
            }
        }
    } else {
        double bw = 0, bb = 0;
        for (const FeedImage &im : imgs) {
            const double m = (double)im.w * im.h;
            if (kind == SB_BLEND_FEATHER) bw += m * (1 + 4 + 4 + 4 + 4), bb += 4 * m;  // DT passes; weight read
            bb += l0 * m;
        }
        bb += 4.0 * (double)roi.w * roi.h;
        if (kind == SB_BLEND_FEATHER) v.emplace_back("feather_weights", bw);
        v.emplace_back(kind == SB_BLEND_FEATHER ? "feather_blend" : "no_blend", bb);
    }
    return v;
}

double BlendPlan::model_bytes(double *pyr, double *collapse) const
{
    double bp = 0, bc = 0;
    for (const auto &kv : launch_bytes()) {
        if (kv.first.rfind("pyrdown", 0) == 0 || kv.first == "feather_weights") bp += kv.second;
        else bc += kv.second;
    }
    if (pyr) *pyr = bp;
    if (collapse) *collapse = bc;
    return bp + bc;
}

}  // namespace sb
