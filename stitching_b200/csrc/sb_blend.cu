// sb_blend.cu -- the blend half of the hot path.
//
// multiband (stitching/blender.py:30-32, :41, :46 -> cv.detail_MultiBandBlender):
//   one kernel per pyramid level, coarse to fine, over the padded panorama.  Per pixel it does, for the
//   fed images covering it IN FEED ORDER:  L = G_l - pyrUp(G_{l+1}) (saturating; L = G_nb at the top),
//   acc += (short)trunc(L * W_l) (wrap-around int16), wsum += W_l;  then the blend step
//   n = (short)trunc(acc / (wsum + 1e-5)) and the collapse  C_l = sat16(pyrUp(C_{l+1}) + n).
//   The reference's accumulators (dst_pyr_laplace / dst_band_weights) therefore never exist in memory:
//   int16 wrap-around adds are associative and the float adds happen in the same order as
//   MultiBandBlender::feed performs them, so the result is identical to eager per-feed accumulation.
//   At level 0 the kernel also applies `dst_mask = wsum > 1e-5`, zeroes outside it, crops to the
//   unpadded roi and fuses cv.convertScaleAbs (blender.py:47).
//
// feather / no (blender.py:27-28, 34-36 -> cv.detail_FeatherBlender, cv.detail.Blender): single level.
#include "sb_launch.h"
#include "sb_gather.cuh"

namespace sb {

namespace {

constexpr int CL_BX = 32, CL_BY = 8;

// simple variant: one thread per pano pixel of level l, loops over all images with a rect test
__global__ void __launch_bounds__(CL_BX *CL_BY)
    k_collapse_gather(const FeedImage *__restrict__ imgs, int n, const PanoLevel *__restrict__ pano, int l, int nb, int lw,
                      int lh, PanoOut out)
{
    const int x = blockIdx.x * CL_BX + threadIdx.x;
    const int y = blockIdx.y * CL_BY + threadIdx.y;
    if (x >= lw || y >= lh) return;
    if (l == 0 && (x >= out.w || y >= out.h)) return;  // level 0 is the last step: the pad is never read

    collapse_pixel(imgs, n, pano, l, nb, x, y, out);
}

// feather / no: one thread per pano pixel, images in feed order
__global__ void __launch_bounds__(CL_BX *CL_BY) k_simple_blend(const FeedImage *__restrict__ imgs, int n, int feather, PanoOut out)
{
#ifndef SB_EMU
    // the images whose rect touches this 32x8 tile, in feed order: warp 0 compacts them into shared memory (with sixteen
    // images a pixel is covered by two or three: the per-pixel loop over all of them was most of the kernel)
    __shared__ unsigned short list[SB_MAX_IMAGES];
    __shared__ int list_n;
    if (threadIdx.y == 0) {
        const int tx0 = blockIdx.x * CL_BX, ty0 = blockIdx.y * CL_BY;
        int cnt = 0;
        for (int base = 0; base < n; base += 32) {
            const int i = base + threadIdx.x;
            bool c = false;
            if (i < n) {
                const FeedImage &im = imgs[i];
                c = tx0 < im.dx + im.w && tx0 + CL_BX > im.dx && ty0 < im.dy + im.h && ty0 + CL_BY > im.dy;
            }
            const unsigned m = __ballot_sync(0xffffffffu, c);
            if (c) list[cnt + __popc(m & ((1u << threadIdx.x) - 1u))] = (unsigned short)i;
            cnt += __popc(m);
        }
        if (threadIdx.x == 0) list_n = cnt;
    }
    __syncthreads();
    const int n_cover = list_n;
#endif
    const int x = blockIdx.x * CL_BX + threadIdx.x;
    const int y = blockIdx.y * CL_BY + threadIdx.y;
    if (x >= out.w || y >= out.h) return;
    int acc[3] = {0, 0, 0};
    float wsum = 0.f;
    unsigned mor = 0;
#ifndef SB_EMU
    for (int k = 0; k < n_cover; ++k) {
        const FeedImage &im = imgs[list[k]];
#else
    for (int i = 0; i < n; ++i) {
        const FeedImage &im = imgs[i];
#endif
        const int X = x - im.dx, Y = y - im.dy;
        if ((unsigned)X >= (unsigned)im.w || (unsigned)Y >= (unsigned)im.h) continue;
        int g[3];
        unsigned m;
        if (im.rgbm) {
            const unsigned p = __ldg(im.rgbm + (long long)Y * im.rgbm_pitch + X);
            g[0] = p & 255u; g[1] = (p >> 8) & 255u; g[2] = (p >> 16) & 255u; m = p >> 24;
        } else {
            const int16_t *q = im.s16 + (long long)Y * im.s16_pitch + (long long)X * 3;
            g[0] = q[0]; g[1] = q[1]; g[2] = q[2];
            m = im.mask[(long long)Y * im.mask_pitch + X];
        }
        if (feather) {
            const float wt = im.fw[(long long)Y * im.w + X];
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[c] += f2s_wrap(fmul((float)g[c], wt));
            wsum = fadd(wsum, wt);
        } else {
            if (m) { acc[0] = g[0]; acc[1] = g[1]; acc[2] = g[2]; }
            mor |= m;
        }
    }
    int v[3];
    bool on;
    unsigned mv;
    if (feather) {
        // one refined reciprocal serves the three channels (sb_device.cuh: 1e-5 <= den <= 256, |a| <= 32768: inside the
        // ranges where the shortcut equals the IEEE division)
        const float den = fadd(wsum, SB_WEIGHT_EPS), rr = rcp_refined(den);
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = f2s_wrap(fdiv_by((float)(short)acc[c], den, rr));
        on = wsum > SB_WEIGHT_EPS;
        mv = on ? 255u : 0u;
    } else {
        v[0] = acc[0]; v[1] = acc[1]; v[2] = acc[2];
        on = mor != 0;
        mv = mor;
    }
    store_final(out, x, y, v, on, mv);
}

// sharded feather blend (SURVEY 8e for BASELINE configs[4]): the same per-pixel arithmetic over a region of the pano,
// with the partial sums of other ranks as additional items -- int16 wrap-around adds are exact under any grouping, the
// float weight sums are grouped per rank (see sb_shard.cpp)
__global__ void __launch_bounds__(CL_BX *CL_BY) k_feather_region(const __grid_constant__ FeatherRegionArgs A)
{
    const int x = A.rx0 + blockIdx.x * CL_BX + threadIdx.x;
    const int y = A.ry0 + blockIdx.y * CL_BY + threadIdx.y;
    if (x >= A.rx0 + A.rw || y >= A.ry0 + A.rh) return;
    int acc[3] = {0, 0, 0};
    float wsum = 0.f;
    auto add_slab = [&](const FeatherSlab &S) {
        const int X = x - S.x0, Y = y - S.y0;
        if ((unsigned)X >= (unsigned)S.w || (unsigned)Y >= (unsigned)S.h) return;
        const int o = Y * S.pitch + X;
        acc[0] += S.acc[o];
        acc[1] += S.acc[S.plane + o];
        acc[2] += S.acc[2 * S.plane + o];
        wsum = fadd(wsum, S.wsum[o]);
    };
    for (int k = 0; k < A.n_before; ++k) add_slab(A.slabs[k]);
    for (int i = A.i0; i < A.i1; ++i) {
        const FeedImage &im = A.imgs[i];
        const int X = x - im.dx, Y = y - im.dy;
        if ((unsigned)X >= (unsigned)im.w || (unsigned)Y >= (unsigned)im.h) continue;
        int g[3];
        if (im.rgbm) {
            const unsigned p = __ldg(im.rgbm + (long long)Y * im.rgbm_pitch + X);
            g[0] = p & 255u; g[1] = (p >> 8) & 255u; g[2] = (p >> 16) & 255u;
        } else {
            const int16_t *q = im.s16 + (long long)Y * im.s16_pitch + (long long)X * 3;
            g[0] = q[0]; g[1] = q[1]; g[2] = q[2];
        }
        const float wt = im.fw[(long long)Y * im.w + X];
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += f2s_wrap(fmul((float)g[c], wt));
        wsum = fadd(wsum, wt);
    }
    for (int k = 0; k < A.n_after; ++k) add_slab(A.slabs[A.n_before + k]);
    if (A.partial) {
        const int o = (y - A.ry0) * A.slab_pitch + (x - A.rx0);
        A.slab_acc[o] = (int16_t)acc[0];
        A.slab_acc[A.slab_plane + o] = (int16_t)acc[1];
        A.slab_acc[2 * A.slab_plane + o] = (int16_t)acc[2];
        A.slab_w[o] = wsum;
        return;
    }
    const float den = fadd(wsum, SB_WEIGHT_EPS), rr = rcp_refined(den);
    int v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = f2s_wrap(fdiv_by((float)(short)acc[c], den, rr));
    const bool on = wsum > SB_WEIGHT_EPS;
    store_final(A.out, x - A.out_x0, y - A.out_y0, v, on, on ? 255u : 0u);
}

// ---- feather weights: w = min(L1 distance to the nearest zero mask pixel * sharpness, 1) ------------
// exact city-block distance = min over rows of (row distance + |dy|): a row pass then a column pass,
// each a forward and a backward min-plus sweep.  "no zero pixel" stays at DT_INF -> weight 1.
#define DT_INF (1 << 29)

__device__ __forceinline__ unsigned mask_at(const FeedImage &im, int x, int y)
{
    if (im.rgbm) return __ldg(im.rgbm + (long long)y * im.rgbm_pitch + x) >> 24;
    return im.mask[(long long)y * im.mask_pitch + x];
}

// one thread per row: distance along the row to the nearest zero (int stored in the float buffer's bits)
__global__ void k_dt_rows(const FeedImage *__restrict__ imgs, int i)
{
    const FeedImage &im = imgs[i];
    const int y = blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= im.h) return;
    int *d = (int *)im.fw + (long long)y * im.w;
    int run = DT_INF;
    for (int x = 0; x < im.w; ++x) {
        run = mask_at(im, x, y) ? min(run + 1, DT_INF) : 0;
        d[x] = run;
    }
    run = DT_INF;
    for (int x = im.w - 1; x >= 0; --x) {
        run = d[x] == 0 ? 0 : min(run + 1, DT_INF);
        d[x] = min(d[x], run);
    }
}
// one thread per column: vertical min-plus sweeps, then the weight
__global__ void k_dt_cols(const FeedImage *__restrict__ imgs, int i, float sharpness)
{
    const FeedImage &im = imgs[i];
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= im.w) return;
    int *d = (int *)im.fw;
    int run = DT_INF;
    for (int y = 0; y < im.h; ++y) {
        run = min(d[(long long)y * im.w + x], min(run + 1, DT_INF));
        d[(long long)y * im.w + x] = run;
    }
    run = DT_INF;
    float *f = (float *)im.fw;
    for (int y = im.h - 1; y >= 0; --y) {
        run = min(d[(long long)y * im.w + x], min(run + 1, DT_INF));
        const float dist = run >= DT_INF ? 3.402823466e+38f : (float)run;
        f[(long long)y * im.w + x] = fminf(fmul(dist, sharpness), 1.f);
    }
}


}  // namespace

int launch_collapse_gather(const FeedImage *imgs_dev, int n, const PanoLevel *pano_dev, int l, int nb, int lw, int lh, PanoOut out,
                           cudaStream_t s)
{
    int gw = l == 0 ? out.w : lw, gh = l == 0 ? out.h : lh;
    if (gw <= 0 || gh <= 0) return SB_OK;
    dim3 block(CL_BX, CL_BY), grid(div_up(gw, CL_BX), div_up(gh, CL_BY));
    launch(k_collapse_gather, grid, block, 0, s, imgs_dev, n, pano_dev, l, nb, lw, lh, out);
    return launch_check("k_collapse_gather");
}

int launch_feather_weights_fast(const FeedImage *imgs_dev, const FeedImage *imgs_host, int n, float sharpness, cudaStream_t s);

int launch_feather_weights(const FeedImage *imgs_dev, const FeedImage *imgs_host, int n, float sharpness, cudaStream_t s)
{
    bool fast = !use_simple_kernels();
#ifdef SB_EMU
    if (!getenv("SB_EMU_LANES")) fast = false;  // the ballot-based row kernel needs the (slow) lane emulation: on request only
#endif
    if (fast) return launch_feather_weights_fast(imgs_dev, imgs_host, n, sharpness, s);
    for (int i = 0; i < n; ++i) {
        launch(k_dt_rows, dim3(div_up(imgs_host[i].h, 64)), dim3(64), 0, s, imgs_dev, i);
        launch(k_dt_cols, dim3(div_up(imgs_host[i].w, 64)), dim3(64), 0, s, imgs_dev, i, sharpness);
    }
    return launch_check("k_dt");
}

int launch_feather_region(const FeatherRegionArgs &A, cudaStream_t s)
{
    if (A.rw <= 0 || A.rh <= 0) return SB_OK;
    dim3 block(CL_BX, CL_BY), grid(div_up(A.rw, CL_BX), div_up(A.rh, CL_BY));
    launch(k_feather_region, grid, block, 0, s, A);
    return launch_check("k_feather_region");
}

int launch_simple_blend(const FeedImage *imgs_dev, int n, int feather, PanoOut out, cudaStream_t s)
{
    if (out.w <= 0 || out.h <= 0) return SB_OK;
    dim3 block(CL_BX, CL_BY), grid(div_up(out.w, CL_BX), div_up(out.h, CL_BY));
    launch(k_simple_blend, grid, block, 0, s, imgs_dev, n, feather, out);
    return launch_check("k_simple_blend");
}

}  // namespace sb
