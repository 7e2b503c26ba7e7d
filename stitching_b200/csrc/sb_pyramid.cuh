// sb_pyramid.cuh -- per-pixel accessors and filter taps of the multiband pyramids (device).
//
// Semantics restated from cv::pyrDown / cv::pyrUp / copyMakeBorder as MultiBandBlender::feed uses them
// (reached from stitching/blender.py:41):
//   level 0 of a fed image is the image extended to its padded rect: BORDER_REFLECT for the colours,
//   constant 0 for the weight (mask/255);   pyrDown: 5x5 [1 4 6 4 1]^2, BORDER_REFLECT_101 at the padded
//   rect's edge, int16 (s+128)>>8, float *(1/256);   pyrUp to exactly 2x: left/top reflect-101,
//   right/bottom replicate, (s+32)>>6.
#pragma once
#include "sb_device.cuh"
#include "sb_internal.h"

namespace sb {

// float(1./255.): MultiBandBlender converts the mask with convertTo(CV_32F, 1./255.) = float(m) * float(alpha)
#define SB_INV255 0.0039215688593685626983642578125f

// level-0 sample at padded-rect coordinates (X, Y), both already inside [0,pw) x [0,ph)
__device__ __forceinline__ void load_level0(const FeedImage &im, int X, int Y, int c[3], float &wt)
{
    const int ix = X - im.left, iy = Y - im.top;
    const bool inside = (unsigned)ix < (unsigned)im.w && (unsigned)iy < (unsigned)im.h;
    const int sx = reflect(ix, im.w), sy = reflect(iy, im.h);
    unsigned m;
    if (im.rgbm) {
        const unsigned p = __ldg(im.rgbm + (long long)sy * im.rgbm_pitch + sx);
        c[0] = p & 255u;
        c[1] = (p >> 8) & 255u;
        c[2] = (p >> 16) & 255u;
        m = p >> 24;
    } else {
        const int16_t *q = im.s16 + (long long)sy * im.s16_pitch + (long long)sx * 3;
        c[0] = q[0];
        c[1] = q[1];
        c[2] = q[2];
        m = im.mask[(long long)sy * im.mask_pitch + sx];
    }
    wt = inside ? fmul((float)m, SB_INV255) : 0.f;
}

// the three colours of element o of a level >= 1, either layout (sb_internal.h: one word per pixel or planar int16)
__device__ __forceinline__ void load_colours(const Level &L, long long o, int c[3])
{
    if (L.q) {
        const unsigned v = L.q[o];
        c[0] = (int)(v & 255u);
        c[1] = (int)((v >> 8) & 255u);
        c[2] = (int)(v >> 16);
    } else {
        c[0] = L.g[o];
        c[1] = L.g[L.plane + o];
        c[2] = L.g[2 * L.plane + o];
    }
}
__device__ __forceinline__ void store_colours(const Level &L, long long o, const int c[3])
{
    if (L.q) {
        L.q[o] = (unsigned)c[0] | ((unsigned)c[1] << 8) | ((unsigned)c[2] << 16);  // bytes: see sb_internal.h
    } else {
        L.g[o] = (int16_t)c[0];
        L.g[L.plane + o] = (int16_t)c[1];
        L.g[2 * L.plane + o] = (int16_t)c[2];
    }
}

// sample of level l (l >= 0) at level-rect coordinates (X, Y) inside the level
__device__ __forceinline__ void load_level(const FeedImage &im, int l, int X, int Y, int c[3], float &wt)
{
    if (l == 0) {
        load_level0(im, X, Y, c, wt);
        return;
    }
    const Level &L = im.lv[l];
    const long long o = (long long)Y * L.pitch + X;
    load_colours(L, o, c);
    wt = L.w[o];
}

// colours only
__device__ __forceinline__ void load_level_rgb(const FeedImage &im, int l, int X, int Y, int c[3])
{
    if (l == 0) {
        float wt;
        load_level0(im, X, Y, c, wt);
        return;
    }
    const Level &L = im.lv[l];
    load_colours(L, (long long)Y * L.pitch + X, c);
}

// pyrUp tap geometry along one axis for destination index d of a 2x upsample of n samples:
// source indices (prev, cur, next) and integer weights; even d: 1,6,1; odd d: 0,4,4
struct UpTap {
    int ip, ic, in;
    int wp, wc, wn;
};
__device__ __forceinline__ UpTap up_tap(int d, int n)
{
    UpTap t;
    t.ic = d >> 1;
    t.ip = t.ic > 0 ? t.ic - 1 : (n > 1 ? 1 : 0);
    t.in = t.ic + 1 < n ? t.ic + 1 : n - 1;
    if (d & 1) {
        t.wp = 0; t.wc = 4; t.wn = 4;
    } else {
        t.wp = 1; t.wc = 6; t.wn = 1;
    }
    return t;
}

// pyrUp of one int16 plane S (sw x sh) evaluated at destination pixel (x, y): (sum + 32) >> 6
__device__ __forceinline__ int pyrup_at(const int16_t *__restrict__ S, int pitch, int sw, int sh, int x, int y)
{
    const UpTap tx = up_tap(x, sw), ty = up_tap(y, sh);
    const int16_t *rp = S + (long long)ty.ip * pitch, *rc = S + (long long)ty.ic * pitch, *rn = S + (long long)ty.in * pitch;
    const int hp = tx.wp * rp[tx.ip] + tx.wc * rp[tx.ic] + tx.wn * rp[tx.in];
    const int hc = tx.wp * rc[tx.ip] + tx.wc * rc[tx.ic] + tx.wn * rc[tx.in];
    const int hn = tx.wp * rn[tx.ip] + tx.wc * rn[tx.ic] + tx.wn * rn[tx.in];
    return (ty.wp * hp + ty.wc * hc + ty.wn * hn + 32) >> 6;
}

// the same for the three colours of a fed image's level (either layout), destination pixel (x, y) of level l
__device__ __forceinline__ void pyrup_level_at(const Level &U, int sw, int sh, int x, int y, int out[3])
{
    const UpTap tx = up_tap(x, sw), ty = up_tap(y, sh);
    const int xs[3] = {tx.ip, tx.ic, tx.in}, xw[3] = {tx.wp, tx.wc, tx.wn};
    const int ys[3] = {ty.ip, ty.ic, ty.in}, yw[3] = {ty.wp, ty.wc, ty.wn};
    int acc[3] = {0, 0, 0};
    for (int j = 0; j < 3; ++j) {
        int h[3] = {0, 0, 0};
        for (int i = 0; i < 3; ++i) {
            int c[3];
            load_colours(U, (long long)ys[j] * U.pitch + xs[i], c);
            for (int k = 0; k < 3; ++k) h[k] += xw[i] * c[k];
        }
        for (int k = 0; k < 3; ++k) acc[k] += yw[j] * h[k];
    }
    for (int k = 0; k < 3; ++k) out[k] = (acc[k] + 32) >> 6;
}

// float 5-tap [1 4 6 4 1] with the two summation orders of the reference build (4-lane SSE body vs scalar
// borders/tails); `simd` selects the order
__device__ __forceinline__ float tap5_h(float s0, float s1, float s2, float s3, float s4, bool simd)
{
    const float m6 = fmul(s2, 6.f), m4 = fmul(fadd(s1, s3), 4.f);
    return simd ? fadd(m6, fadd(m4, fadd(s0, s4))) : fadd(fadd(fadd(m6, m4), s0), s4);
}
__device__ __forceinline__ float tap5_v(float r0, float r1, float r2, float r3, float r4, bool simd)
{
    const float v = simd ? fadd(fmul(fadd(fadd(r1, r3), r2), 4.f), fadd(fadd(r0, r4), fadd(r2, r2)))
                         : fadd(fadd(fadd(fmul(r2, 6.f), fmul(fadd(r1, r3), 4.f)), r0), r4);
    return fmul(v, 0.00390625f);
}
// first output column that is NOT in the horizontal SIMD body [1, hs_end) for a source row of W floats
__host__ __device__ __forceinline__ int pyrdown_hs_end(int W)
{
    const int dw = (W + 1) / 2;
    int width0 = (W - 3) / 2 + 1;
    if (width0 > dw) width0 = dw;
    return width0 >= 5 ? 1 + ((width0 - 1) / 4) * 4 : 1;
}

}  // namespace sb
