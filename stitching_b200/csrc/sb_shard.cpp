// sb_shard.cpp -- geometry and launch sequencing of the multi-GPU composite (no reference counterpart: the
// reference is single-process; this is SURVEY.md 8(e)).
//
// Images are dealt to ranks in contiguous blocks (feed order is rank order); the padded panorama is cut into
// column strips, one per rank, at multiples of 2^nb.  A rank computes warp + pyramids for its own images only.
// Where the padded footprint of its images reaches into another rank's strip it hands that rank a SLAB per level:
// its partial sums (acc int16x3 with wrap-around, wsum float32) over the part of the strip -- plus a 2-pixel
// margin per level, which is what the pyrUp of the next finer level reads -- that its footprint covers.  The owner
// adds the slabs and its own images in rank order inside the ordinary per-level kernel and collapses its strip.
// int16 wrap-around sums are exact under any grouping; the float weight sums are grouped per rank (each slab a sum
// from 0, added in rank order around the owner's own images), which can differ from the single-GPU order by float
// re-association.  The grouping is deterministic: tests/shard_fuzz.py restates it with the CPU oracle
// (oracle.Blender.fold) and the tests compare every strip with it bit for bit.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "sb_shard.h"

namespace sb {

namespace {
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
}

// Feather (single level): rank `src` hands rank `dst` its partial sums over (bounding box of its images) x (dst's strip).
void ShardPlan::feather_slab_geometry(const BlendPlan &plan, int src, int dst, PeerSlab *ps) const
{
    int f0, fc;
    block_of((int)plan.imgs.size(), world, src, &f0, &fc);
    std::memset(ps->lv, 0, sizeof ps->lv);
    ps->bytes = ps->split = 0;
    int x0 = 1 << 30, y0 = 1 << 30, x1 = -1, y1 = -1;
    for (int i = f0; i < f0 + fc; ++i) {
        const FeedImage &im = plan.imgs[i];
        x0 = std::min(x0, im.dx);
        y0 = std::min(y0, im.dy);
        x1 = std::max(x1, im.dx + im.w);
        y1 = std::max(y1, im.dy + im.h);
    }
    const int q = reversed ? world - 1 - dst : dst;  // dst's place in the spatial order of the strips
    if (axis == 0) {
        x0 = std::max(x0, bounds[q]);
        x1 = std::min(x1, bounds[q + 1]);
    } else {
        y0 = std::max(y0, bounds[q]);
        y1 = std::min(y1, bounds[q + 1]);
    }
    if (fc == 0 || x1 <= x0 || y1 <= y0) return;
    SlabLevel &L = ps->lv[0];
    L.x0 = x0;
    L.y0 = y0;
    L.w = x1 - x0;
    L.h = y1 - y0;
    L.pitch = (int)align_up((size_t)L.w, 8);
    L.plane = L.pitch * L.h;
    L.acc_off = 0;
    L.w_off = align_up((size_t)3 * L.plane * sizeof(int16_t), 256);
    ps->bytes = ps->split = align_up(L.w_off + (size_t)L.plane * sizeof(float), 256);  // everything travels as "part 0"
}

void ShardPlan::slab_geometry(const BlendPlan &plan, int src, int dst, PeerSlab *ps) const
{
    if (plan.kind == SB_BLEND_FEATHER) {
        feather_slab_geometry(plan, src, dst, ps);
        return;
    }
    int f0, fc;
    block_of((int)plan.imgs.size(), world, src, &f0, &fc);
    size_t off = 0;
    std::memset(ps->lv, 0, sizeof ps->lv);
    ps->split = 0;
    for (int l = 0; l <= plan.nb; ++l) {
        SlabLevel &L = ps->lv[l];
        if (fc == 0) continue;
        // Bounding box of where the source rank's weights can be non-zero at this level.  W_0 is non-zero only inside
        // the fed image's own rect (the padding is a constant-0 border); every pyrDown grows that support by at most
        // 2 samples per side, i.e. it stays within 3 level-l pixels of the scaled image rect.  Outside it the partial
        // sums are exactly (acc, wsum) = (0, 0) and need not travel.  Clipped to the padded footprint, kept even.
        int fx0 = 1 << 30, fy0 = 1 << 30, fx1 = -1, fy1 = -1;
        const int even = l < plan.nb ? ~1 : ~0;
        for (int i = f0; i < f0 + fc; ++i) {
            const FeedImage &im = plan.imgs[i];
            const int X0 = im.px + im.left, Y0 = im.py + im.top, X1 = X0 + im.w, Y1 = Y0 + im.h;
            const int px0 = im.px >> l, py0 = im.py >> l, px1 = (im.px + im.pw) >> l, py1 = (im.py + im.ph) >> l;
            fx0 = std::min(fx0, std::max(px0, ((X0 >> l) - 3) & even));
            fy0 = std::min(fy0, std::max(py0, ((Y0 >> l) - 3) & even));
            fx1 = std::max(fx1, std::min(px1, ((((X1 - 1) >> l) + 4) + 1) & even));
            fy1 = std::max(fy1, std::min(py1, ((((Y1 - 1) >> l) + 4) + 1) & even));
        }
        int a, b;
        plan.region_x(bounds[dst], bounds[dst + 1], l, &a, &b);
        const int x0 = std::max(a, fx0), x1 = std::min(b, fx1);
        if (x1 <= x0 || fy1 <= fy0) continue;
        L.x0 = x0;
        L.y0 = fy0;
        L.w = x1 - x0;
        L.h = fy1 - fy0;
        L.pitch = (int)align_up((size_t)L.w, 8);
        L.plane = L.pitch * L.h;
        L.acc_off = off;
        off = align_up(off + (size_t)3 * L.plane * sizeof(int16_t), 256);
        L.w_off = off;
        off = align_up(off + (size_t)L.plane * sizeof(float), 256);
        if (l == 0) ps->split = off;
    }
    ps->bytes = off;
}

int ShardPlan::build(const BlendPlan &plan, int rank_, int world_)
{
    const int n = (int)plan.imgs.size();
    if (!(plan.kind == SB_BLEND_FEATHER || (plan.kind == SB_BLEND_MULTIBAND && plan.nb >= 1))) {
        set_error("sharded composite: needs the feather blender or the multiband blender with at least one band (got kind %d, %d bands)",
                  plan.kind, plan.nb);
        return SB_ERR_INVALID;
    }
    if (world_ < 1 || rank_ < 0 || rank_ >= world_ || n < world_) {
        set_error("sharded composite: rank %d of %d with %d images", rank_, world_, n);
        return SB_ERR_INVALID;
    }
    rank = rank_;
    world = world_;
    feather = plan.kind == SB_BLEND_FEATHER;
    axis = 0;
    reversed = false;
    block_of(n, world, rank, &first, &count);
    SB_TRY(feather ? feather_bounds(plan) : multiband_bounds(plan));
    send.assign(world, PeerSlab());
    recv.assign(world, PeerSlab());
    for (int p = 0; p < world; ++p) {
        if (p == rank) continue;
        slab_geometry(plan, rank, p, &send[p]);
        slab_geometry(plan, p, rank, &recv[p]);
    }
    return SB_OK;
}

int ShardPlan::multiband_bounds(const BlendPlan &plan)
{
    const int n = (int)plan.imgs.size();
    // strip boundaries: halfway between the centres of the neighbouring blocks' edge images, snapped to 2^nb.  Blocks
    // that run right to left would give decreasing boundaries: refused rather than clamped, which would leave one rank
    // the whole panorama and the others nothing.  Equal boundaries (an empty strip) are fine.
    const int a = 1 << plan.nb;
    bounds.assign(world + 1, 0);
    bounds[world] = plan.wp;
    for (int r = 1; r < world; ++r) {
        int f0, fc, g0, gc;
        block_of(n, world, r - 1, &f0, &fc);
        block_of(n, world, r, &g0, &gc);
        const FeedImage &L = plan.imgs[f0 + fc - 1], &R = plan.imgs[g0];
        const long long mid = ((long long)L.px + L.left + L.w / 2 + R.px + R.left + R.w / 2) / 2;
        const int b = (int)std::min<long long>((mid + a / 2) / a * a, plan.wp);
        if (b < bounds[r - 1]) {
            set_error("sharded composite: image blocks are not ordered left to right in the panorama (boundary %d at column %d, "
                      "boundary %d at column %d)", r - 1, bounds[r - 1], r, b);
            return SB_ERR_INVALID;
        }
        bounds[r] = b;
    }
    return SB_OK;
}

// Feather: the image blocks are either side by side (a yaw ring: column strips) or stacked (the rows of an affine grid,
// BASELINE configs[4]: row strips); the strip boundaries lie halfway between the neighbouring blocks' bounding boxes.
int ShardPlan::feather_bounds(const BlendPlan &plan)
{
    const int n = (int)plan.imgs.size();
    std::vector<double> cx(world), cy(world);
    std::vector<int> lo_x(world), hi_x(world), lo_y(world), hi_y(world);
    for (int r = 0; r < world; ++r) {
        int f0, fc;
        block_of(n, world, r, &f0, &fc);
        int x0 = 1 << 30, y0 = 1 << 30, x1 = -1, y1 = -1;
        for (int i = f0; i < f0 + fc; ++i) {
            const FeedImage &im = plan.imgs[i];
            x0 = std::min(x0, im.dx); y0 = std::min(y0, im.dy);
            x1 = std::max(x1, im.dx + im.w); y1 = std::max(y1, im.dy + im.h);
        }
        lo_x[r] = x0; hi_x[r] = x1; lo_y[r] = y0; hi_y[r] = y1;
        cx[r] = 0.5 * (x0 + x1);
        cy[r] = 0.5 * (y0 + y1);
    }
    // the blocks follow each other along x or y, in either direction (an affine grid whose rows run bottom to top in the
    // panorama is as good as one running top to bottom); prefer the axis along which they are spread further apart
    bool inc_x = true, inc_y = true, dec_x = true, dec_y = true;
    for (int r = 1; r < world; ++r) {
        inc_x = inc_x && cx[r] > cx[r - 1];
        dec_x = dec_x && cx[r] < cx[r - 1];
        inc_y = inc_y && cy[r] > cy[r - 1];
        dec_y = dec_y && cy[r] < cy[r - 1];
    }
    const bool mono_x = inc_x || dec_x, mono_y = inc_y || dec_y;
    if (!mono_x && !mono_y) {
        set_error("sharded composite: image blocks are ordered neither along x nor along y in the panorama (block centres (%.1f, %.1f) .. (%.1f, %.1f))",
                  cx[0], cy[0], cx[world - 1], cy[world - 1]);
        return SB_ERR_INVALID;
    }
    axis = (mono_y && (!mono_x || std::fabs(cy[world - 1] - cy[0]) > std::fabs(cx[world - 1] - cx[0]))) ? 1 : 0;
    reversed = axis == 0 ? !inc_x : !inc_y;
    const int extent = axis == 0 ? plan.roi.w : plan.roi.h;
    bounds.assign(world + 1, 0);  // in spatial order: the strip of rank r is [bounds[q], bounds[q + 1]), q = reversed ? world-1-r : r
    bounds[world] = extent;
    for (int q = 1; q < world; ++q) {
        const int ra = reversed ? world - q : q - 1, rb = reversed ? world - 1 - q : q;  // the ranks at places q-1 and q
        const int a = axis == 0 ? hi_x[ra] : hi_y[ra], b = axis == 0 ? lo_x[rb] : lo_y[rb];
        int m = (a + b) / 2;  // middle of the overlap (or of the gap) between the two blocks
        m = std::max(m, bounds[q - 1]);
        bounds[q] = std::min(m, extent);
    }
    return SB_OK;
}

void ShardPlan::strip(const BlendPlan &plan, int *lo, int *hi) const
{
    const int extent = axis == 0 ? plan.roi.w : plan.roi.h;
    const int q = reversed ? world - 1 - rank : rank;
    *lo = std::min(bounds[q], extent);
    *hi = std::min(bounds[q + 1], extent);
}

int ShardPlan::allocate(const BlendPlan &plan, cudaStream_t s)
{
    release(s);
    const int n = (int)plan.imgs.size();
    SB_CUDA(cudaStreamCreateWithFlags(&comm_, cudaStreamNonBlocking));
    for (int k = 0; k < 2; ++k) {
        SB_CUDA(cudaEventCreateWithFlags(&e_part_[k], cudaEventDisableTiming));
        SB_CUDA(cudaEventCreateWithFlags(&e_xchg_[k], cudaEventDisableTiming));
    }
    SB_TRY(connect(plan, s));  // direct exchange over NVLink when the ranks can map each other's memory (sb_peer.cpp)
    for (int p = 0; p < world; ++p) {
        if (send[p].bytes) SB_TRY(dev_alloc(&send[p].buf, send[p].bytes, s));
        if (!recv[p].bytes) continue;
        if (connected)
            recv[p].buf = (char *)arena + recv_off[p];
        else
            SB_TRY(dev_alloc(&recv[p].buf, recv[p].bytes, s));
    }
    if (feather) {
        // the slabs this rank receives, lower ranks first
        std::vector<FeatherSlab> fs;
        feather_before_ = feather_after_ = 0;
        for (int p = 0; p < world; ++p) {
            const SlabLevel &L = recv[p].lv[0];
            if (p == rank || !recv[p].bytes || L.w == 0) continue;
            FeatherSlab f;
            f.x0 = L.x0; f.y0 = L.y0; f.w = L.w; f.h = L.h; f.pitch = L.pitch; f.plane = L.plane;
            f.acc = (const int16_t *)((const char *)recv[p].buf + L.acc_off);
            f.wsum = (const float *)((const char *)recv[p].buf + L.w_off);
            fs.push_back(f);
            (p < rank ? feather_before_ : feather_after_)++;
        }
        SB_TRY(dev_alloc(&feather_items_, std::max<size_t>(fs.size(), 1) * sizeof(FeatherSlab), s));
        if (!fs.empty()) SB_CUDA(cudaMemcpyAsync(feather_items_, fs.data(), fs.size() * sizeof(FeatherSlab), cudaMemcpyHostToDevice, s));
        SB_CUDA(cudaStreamSynchronize(s));
        return SB_OK;
    }
    // item lists per level: slabs of lower ranks, own images, slabs of higher ranks (= feed order)
    std::vector<ColDesc> items;
    std::vector<TileDesc> titems;  // parallel to `items`: the rects the tile kernels test (sb_collapse_tile.cu)
    size_t offs[SB_MAX_BANDS + 2] = {0};
    for (int l = 0; l <= plan.nb; ++l) {
        offs[l] = items.size();
        auto add_slab = [&](int p) {
            const SlabLevel &L = recv[p].lv[l];
            if (!recv[p].bytes || L.w == 0) return;
            ColDesc d;
            std::memset(&d, 0, sizeof d);
            d.ox = L.x0;
            d.oy = L.y0;
            d.w_l = L.w;
            d.h_l = L.h;
            d.g = (const int16_t *)((const char *)recv[p].buf + L.acc_off);
            d.w = (const float *)((const char *)recv[p].buf + L.w_off);
            d.pitch = L.pitch;
            d.plane = L.plane;
            d.kind = 1;
            items.push_back(d);
            TileDesc t;
            std::memset(&t, 0, sizeof t);
            t.x0 = t.ox = L.x0;
            t.y0 = t.oy = L.y0;
            t.w = L.w;
            t.h = L.h;
            titems.push_back(t);
        };
        for (int p = 0; p < rank; ++p) add_slab(p);
        for (int i = first; i < first + count; ++i) {
            items.push_back(plan.col_host[(size_t)l * n + i]);
            titems.push_back(BlendPlan::tile_desc(plan.imgs[i], l));
        }
        for (int p = rank + 1; p < world; ++p) add_slab(p);
        n_items[l] = (int)(items.size() - offs[l]);
        if (n_items[l] > SB_MAX_ITEMS) {
            set_error("sharded composite: %d items at level %d exceed SB_MAX_ITEMS", n_items[l], l);
            return SB_ERR_INVALID;
        }
    }
    SB_TRY(dev_alloc(&items_arena_, std::max<size_t>(items.size(), 1) * sizeof(ColDesc), s));
    if (!items.empty()) SB_CUDA(cudaMemcpyAsync(items_arena_, items.data(), items.size() * sizeof(ColDesc), cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaStreamSynchronize(s));  // `items` is a local
    for (int l = 0; l <= plan.nb; ++l) items_dev[l] = (ColDesc *)items_arena_ + offs[l];
    for (auto &t : tile_items_dev) t = nullptr;
    if (plan.tile_images_ok && !titems.empty()) {
        SB_TRY(dev_alloc(&tile_items_arena_, titems.size() * sizeof(TileDesc), s));
        SB_CUDA(cudaMemcpyAsync(tile_items_arena_, titems.data(), titems.size() * sizeof(TileDesc), cudaMemcpyHostToDevice, s));
        SB_CUDA(cudaStreamSynchronize(s));
        for (int l = 0; l <= plan.nb; ++l) tile_items_dev[l] = (TileDesc *)tile_items_arena_ + offs[l];
    }
    return SB_OK;
}

void ShardPlan::release(cudaStream_t s)
{
    if (comm_) (void)cudaStreamSynchronize(comm_);  // nothing queued there may still use the slabs
    for (auto &p : send) {
        dev_free(p.buf, s);
        p.buf = nullptr;
    }
    for (auto &p : recv) {
        if (!connected) dev_free(p.buf, s);
        p.buf = nullptr;
    }
    if (connected) {
        (void)cudaStreamSynchronize(s);
#ifndef SB_EMU
        for (auto &p : peer_arena)
            if (p) (void)cudaIpcCloseMemHandle(p);
        (void)cudaFree(arena);
#endif
        peer_arena.clear();
        arena = nullptr;
        connected = direct_stores = false;
    }
    dev_free(items_arena_, s);
    items_arena_ = nullptr;
    dev_free(tile_items_arena_, s);
    tile_items_arena_ = nullptr;
    for (auto &t : tile_items_dev) t = nullptr;
    dev_free(feather_items_, s);
    feather_items_ = nullptr;
    if (comm_) (void)cudaStreamDestroy(comm_);
    comm_ = nullptr;
    for (int k = 0; k < 2; ++k) {
        if (e_part_[k]) (void)cudaEventDestroy(e_part_[k]);
        if (e_xchg_[k]) (void)cudaEventDestroy(e_xchg_[k]);
        e_part_[k] = e_xchg_[k] = nullptr;
    }
}

int ShardPlan::partial_out(const BlendPlan &plan, int part, cudaStream_t s)
{
    const int n = (int)plan.imgs.size();
    const int l_lo = part, l_hi = part == 0 ? 0 : plan.nb;  // the part's levels
    for (int p = 0; p < world; ++p) {
        if (p == rank || !send[p].bytes) continue;
        // direct stores: the slab goes straight to its place in the owner's arena (peer stores over NVLink)
        char *dst = direct_stores ? peer_arena[p] + peer_slot[p] : (char *)send[p].buf;
        for (int l = l_lo; l <= l_hi; ++l) {
            const SlabLevel &L = send[p].lv[l];
            if (L.w == 0) continue;
            auto slab = [&](auto &A) {
                std::memset(&A, 0, sizeof A);
                A.rx0 = L.x0;
                A.ry0 = L.y0;
                A.rw = L.w;
                A.rh = L.h;
                A.partial = 1;
                A.slab_acc = (int16_t *)(dst + L.acc_off);
                A.slab_w = (float *)(dst + L.w_off);
                A.slab_pitch = L.pitch;
                A.slab_plane = L.plane;
            };
            if (feather) {
                FeatherRegionArgs A;
                slab(A);
                A.imgs = plan.imgs_dev;
                A.i0 = first;
                A.i1 = first + count;
                SB_TRY(launch_feather_region(A, s));
            } else {
                CollapseArgs A;
                slab(A);
                A.col = plan.col_dev + (size_t)l * n + first;  // this rank's images, contiguous in the level's array
                A.n = count;
                SB_TRY(launch_collapse(A, l, plan.nb, s));
            }
        }
    }
    return SB_OK;
}

int ShardPlan::exchange(int part, cudaStream_t s)
{
    std::vector<int> peers;
    std::vector<void *> sp, rp;
    std::vector<size_t> sb_, rb;
    for (int p = 0; p < world; ++p) {
        if (p == rank || (!send[p].bytes && !recv[p].bytes)) continue;
        size_t s0, s1, r0, r1;
        send[p].part_range(part, &s0, &s1);
        recv[p].part_range(part, &r0, &r1);
        if (s1 == s0 && r1 == r0) continue;
        peers.push_back(p);
        sp.push_back((char *)send[p].buf + s0);
        sb_.push_back(s1 - s0);
        rp.push_back((char *)recv[p].buf + r0);
        rb.push_back(r1 - r0);
    }
    if (peers.empty()) return SB_OK;
    return comm_exchange((int)peers.size(), peers.data(), sp.data(), sb_.data(), rp.data(), rb.data(), s);
}

int ShardPlan::finish(const BlendPlan &plan, const PanoOut &out, int part, cudaStream_t s)
{
    if (feather) {
        int lo, hi;
        strip(plan, &lo, &hi);
        FeatherRegionArgs A;
        std::memset(&A, 0, sizeof A);
        A.imgs = plan.imgs_dev;
        A.i0 = first;
        A.i1 = first + count;
        A.slabs = (const FeatherSlab *)feather_items_;
        A.n_before = feather_before_;
        A.n_after = feather_after_;
        A.rx0 = axis == 0 ? lo : 0;
        A.ry0 = axis == 0 ? 0 : lo;
        A.rw = axis == 0 ? hi - lo : plan.roi.w;
        A.rh = axis == 0 ? plan.roi.h : hi - lo;
        A.out = out;
        A.out_x0 = A.rx0;
        A.out_y0 = A.ry0;
        return launch_feather_region(A, s);
    }
    const int l_lo = part, l_hi = part == 0 ? 0 : plan.nb;  // the part's levels
    for (int l = l_hi; l >= l_lo; --l) {
        CollapseArgs A = plan.collapse_args(l, bounds[rank], bounds[rank + 1], items_dev[l], n_items[l], tile_items_dev[l], out);
        A.has_slabs = n_items[l] > count;  // slabs are items of their own kind in the tile kernels
        SB_TRY(launch_collapse(A, l, plan.nb, s));
    }
    return SB_OK;
}

}  // namespace sb
