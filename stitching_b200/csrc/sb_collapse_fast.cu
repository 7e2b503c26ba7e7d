// sb_collapse_fast.cu -- instruction-lean version of the per-level multiband kernel, all levels.
//
// Same arithmetic as k_collapse_gather (sb_blend.cu; see there for the reference call chain
// stitching/blender.py:41,46 -> MultiBandBlender::feed / ::blend), reorganised for an issue-bound SM, where the
// profile showed the kernel to be issue-bound rather than HBM-bound:
//   * one thread per 2x2 quad: the four pixels share the 3x3 neighbourhood of the coarser level, so each pyrUp
//     (of the image's G_{l+1} and of the collapsed C_{l+1}) is 9 taps per quad, evaluated through shared column sums;
//   * the fed images' levels are one word of bytes per pixel (sb_internal.h), a tap is one 4-byte load: split into
//     lanes after the load, red and blue run as two 16-bit lanes of one word through the pyrUp, the Laplacian and the
//     accumulators (lane-wise VIADD.16x2 = the wrap-around of a short);
//   * compact 16-byte-aligned descriptors (ColDesc) read with vector loads, 32-bit element offsets;
//   * exact early-outs: a fed image whose four weights in the quad are all zero contributes
//     (short)trunc(L * 0) = 0 and wsum + 0 = wsum, i.e. nothing -- at level 0 this is the whole padding ring
//     (constant-0 border of the weight map) and everything outside the warped footprint (mask byte 0);
//   * exact integer forms of the blend division for weight sums 0, 1 and 2, one refined reciprocal per pixel otherwise.
// A block covers a 64x16 tile; warp 0 first compacts the items touching it (in feed order) into shared memory.
//
// Multi-GPU (one rank per GPU, images sharded over ranks): the same kernel runs in two more roles.  An item can
// be a SLAB -- the partial sums (acc int16x3 wrap-around, wsum float32) another rank computed for its own images
// over a rectangle -- which is simply added; and with `partial` set the kernel stops after the accumulation and
// writes such a slab for a neighbour instead of normalising.  A launch covers a REGION of the level (a rank's
// pano strip plus a 2-pixel margin per level, enough for the pyrUp of the next finer level).
#include "sb_launch.h"
#include "sb_pyramid.cuh"

namespace sb {

namespace {

constexpr int CF_BX = 32, CF_BY = 8;
#define SB_WEIGHT_EPS 1e-5f

struct Nbr {  // pyrUp source indices around coarse (ci, cj): element offsets of the three rows, the three columns
    int rp, rc, rn, xp, xc, xn;
};
__device__ __forceinline__ Nbr neighbours(int ci, int cj, int sw, int sh, int pitch)
{
    Nbr q;
    q.xc = ci;
    q.xp = ci > 0 ? ci - 1 : (sw > 1 ? 1 : 0);
    q.xn = ci + 1 < sw ? ci + 1 : sw - 1;
    const int yp = cj > 0 ? cj - 1 : (sh > 1 ? 1 : 0), yn = cj + 1 < sh ? cj + 1 : sh - 1;
    q.rp = yp * pitch;
    q.rc = cj * pitch;
    q.rn = yn * pitch;
    return q;
}
// the four pyrUp values of the quad (u[dy][dx]) from one int16 plane, via vertical column sums:
//   even row: e = a0 + 6 a1 + a2, odd row: o = a1 + a2 (x4 folded into the final shift)
//   (4 s + 32) >> 6 == (s + 8) >> 4 and (16 s + 32) >> 6 == (s + 2) >> 2 for integer s
__device__ __forceinline__ void up_quad(const int16_t *__restrict__ S, const Nbr &q, int u[2][2])
{
    int e[3], o[3];
    const int cols[3] = {q.xp, q.xc, q.xn};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int a0 = __ldg(S + q.rp + cols[k]), a1 = __ldg(S + q.rc + cols[k]), a2 = __ldg(S + q.rn + cols[k]);
        e[k] = a0 + a2 + 6 * a1;
        o[k] = a1 + a2;
    }
    u[0][0] = (e[0] + e[2] + 6 * e[1] + 32) >> 6;
    u[0][1] = (e[1] + e[2] + 8) >> 4;
    u[1][0] = (o[0] + o[2] + 6 * o[1] + 8) >> 4;
    u[1][1] = (o[1] + o[2] + 2) >> 2;
}

// two signed 16-bit lanes in one word
__device__ __forceinline__ unsigned lanes(int lo, int hi) { return ((unsigned)lo & 0xffffu) | ((unsigned)hi << 16); }
__device__ __forceinline__ int lane_lo(unsigned v) { return (int)(short)(v & 0xffffu); }
__device__ __forceinline__ int lane_hi(unsigned v) { return (int)v >> 16; }

// split a colour word r | g << 8 | b << 16 (byte 3 zero) into the lanes r | b << 16 and g
__device__ __forceinline__ unsigned word_rb(unsigned v) { return v & 0x00ff00ffu; }
__device__ __forceinline__ unsigned word_g(unsigned v) { return __byte_perm(v, 0u, 0x4441); }

// The same pyrUp for a fed image's level stored as one word per pixel (r | g << 8 | b << 16): every tap is split into
// the lanes r | b << 16 and g, and red and blue go through the column sums and the final sums as two lanes of one
// word -- the largest intermediate, 64 * 255 + 32, stays below 2^15, so the lanes never meet.  Results:
// u_rb = r | b << 16, u_g = g, each 0..255.
__device__ __forceinline__ void up_quad_lanes(const uint32_t *__restrict__ S, const Nbr &q, unsigned u_rb[2][2], unsigned u_g[2][2])
{
    unsigned e_rb[3], o_rb[3], e_g[3], o_g[3];
    const int cols[3] = {q.xp, q.xc, q.xn};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const unsigned a0 = __ldg(S + q.rp + cols[k]), a1 = __ldg(S + q.rc + cols[k]), a2 = __ldg(S + q.rn + cols[k]);
        e_rb[k] = word_rb(a0) + word_rb(a2) + 6u * word_rb(a1);
        o_rb[k] = word_rb(a1) + word_rb(a2);
        e_g[k] = word_g(a0) + word_g(a2) + 6u * word_g(a1);
        o_g[k] = word_g(a1) + word_g(a2);
    }
    const unsigned M = 0x00ff00ffu;
    u_rb[0][0] = ((e_rb[0] + e_rb[2] + 6u * e_rb[1] + 0x00200020u) >> 6) & M;
    u_rb[0][1] = ((e_rb[1] + e_rb[2] + 0x00080008u) >> 4) & M;
    u_rb[1][0] = ((o_rb[0] + o_rb[2] + 6u * o_rb[1] + 0x00080008u) >> 4) & M;
    u_rb[1][1] = ((o_rb[1] + o_rb[2] + 0x00020002u) >> 2) & M;
    u_g[0][0] = (e_g[0] + e_g[2] + 6u * e_g[1] + 32u) >> 6;
    u_g[0][1] = (e_g[1] + e_g[2] + 8u) >> 4;
    u_g[1][0] = (o_g[0] + o_g[2] + 6u * o_g[1] + 8u) >> 4;
    u_g[1][1] = (o_g[1] + o_g[2] + 2u) >> 2;
}

__device__ __forceinline__ int trunc16(float v) { return (int)(short)__float2int_rz(v); }  // |v| < 2^31 here

// the blend step for one channel: (short)trunc((short)acc / den), x86 cast semantics.  The three channels of a pixel
// share the refined reciprocal of den (sb_device.cuh: the IEEE division's own fast path without its per-quotient range
// check and branch -- the second profile showed the generic division, whose check sends zero numerators to a
// ~100-instruction slow path, to be most of this kernel's instruction stream).  Ranges: den = wsum + 1e-5 lies in
// [2^-17, 2^9], |acc| in [1, 2^15] or acc == 0, which gives exactly 0.
__device__ __forceinline__ int norm16(int acc, float den, float rr)
{
    return f2s_wrap(fdiv_by((float)(int)(short)acc, den, rr));
}

// LV: 0 = level 0 (packed RGBM images), 1 = a middle level, 2 = the top level (no pyrUp anywhere, odd sizes allowed)
template <int LV>
__global__ void __launch_bounds__(CF_BX *CF_BY, 5) k_collapse_fast(const __grid_constant__ CollapseArgs A)
{
    grid_dependency_sync();
    const ColDesc *__restrict__ col = A.col;
    const int n = A.n;
    const int tile_x = A.rx0 + blockIdx.x * (2 * CF_BX), tile_y = A.ry0 + blockIdx.y * (2 * CF_BY);
#ifndef SB_EMU
    // the items whose rect touches this tile, in feed order: warp 0 compacts them into shared memory
    __shared__ unsigned short list[SB_MAX_ITEMS];
    __shared__ int list_n;
    if (threadIdx.y == 0) {
        int cnt = 0;
        for (int base = 0; base < n; base += 32) {
            const int i = base + threadIdx.x;
            bool c = false;
            if (i < n) {
                const int4 r = __ldg(reinterpret_cast<const int4 *>(&col[i].ox));
                c = tile_x < r.x + r.z && tile_x + 2 * CF_BX > r.x && tile_y < r.y + r.w && tile_y + 2 * CF_BY > r.y;
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
    const int x = tile_x + 2 * threadIdx.x, y = tile_y + 2 * threadIdx.y;  // top-left pixel of the quad
    if (x >= A.rx0 + A.rw || y >= A.ry0 + A.rh) return;
    // pixel (dx, dy) of the quad exists?  (only the top level has odd extents)
    bool pv[2][2];
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) pv[dy][dx] = LV != 2 || (x + dx < A.rx0 + A.rw && y + dy < A.ry0 + A.rh);

    // the accumulators (int16 with wrap-around in the reference): red | blue << 16 as two lanes of one word, added
    // with the lane-wise VIADD.16x2 (exactly the wrap-around of a short); green in the low half of an int
    unsigned acc_rb[2][2] = {};
    int acc_g[2][2] = {};
    float wsum[2][2] = {};
#ifndef SB_EMU
    for (int k = 0; k < n_cover; ++k) {
        const ColDesc &d = col[list[k]];
#else
    for (int i = 0; i < n; ++i) {
        const ColDesc &d = col[i];
#endif
        const int4 r = __ldg(reinterpret_cast<const int4 *>(&d.ox));
        const int X = x - r.x, Y = y - r.y;
        bool in[2][2];
        if (LV != 2) {
            // below the top level rect origins and sizes are even: a quad is in or out as a whole
            if ((unsigned)X >= (unsigned)r.z || (unsigned)Y >= (unsigned)r.w) continue;
            in[0][0] = in[0][1] = in[1][0] = in[1][1] = true;
        } else {
            bool any = false;
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    in[dy][dx] = pv[dy][dx] && (unsigned)(X + dx) < (unsigned)r.z && (unsigned)(Y + dy) < (unsigned)r.w;
                    any = any || in[dy][dx];
                }
            if (!any) continue;
        }
        const int4 s1 = __ldg(reinterpret_cast<const int4 *>(&d.top));      // top, pitch, plane, upitch
        const int4 s2 = __ldg(reinterpret_cast<const int4 *>(&d.pad0));     // -, kind, -, -
        if (s2.y == 1) {
            // a slab of partial sums from another rank: add (int16 wrap-around, float in rank order)
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    if (!in[dy][dx]) continue;
                    const int o = (Y + dy) * s1.y + X + dx;
                    acc_rb[dy][dx] = __vadd2(acc_rb[dy][dx], lanes(d.g[o], d.g[2 * s1.z + o]));
                    acc_g[dy][dx] += d.g[s1.z + o];
                    wsum[dy][dx] = fadd(wsum[dy][dx], d.w[o]);
                }
            continue;
        }
        // the level's own colours as lanes: g_rb = r | b << 16, g_g = green (bytes at every level, see sb_internal.h)
        unsigned g_rb[2][2], g_g[2][2];
        float wt[2][2];
        if (LV == 0) {
            const int4 s0 = __ldg(reinterpret_cast<const int4 *>(&d.rgbm_pitch));  // rgbm_pitch, iw, ih, left
            const int ix = X - s0.w, iy = Y - s1.x;
            if (ix + 1 < 0 || ix >= s0.y || iy + 1 < 0 || iy >= s0.z) continue;  // whole quad in the zero-weight padding
            const uint32_t *base = d.rgbm;
            unsigned p[2][2];
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    const bool inside = (unsigned)(ix + dx) < (unsigned)s0.y && (unsigned)(iy + dy) < (unsigned)s0.z;
                    p[dy][dx] = inside ? __ldg(base + (iy + dy) * s0.x + ix + dx) : 0u;
                }
            if (((p[0][0] | p[0][1] | p[1][0] | p[1][1]) >> 24) == 0u) continue;  // all four weights are exactly 0
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    g_rb[dy][dx] = p[dy][dx] & 0x00ff00ffu;
                    g_g[dy][dx] = (p[dy][dx] >> 8) & 255u;
                    wt[dy][dx] = fmul((float)(p[dy][dx] >> 24), SB_INV255);
                }
        } else if (LV == 1) {
            const int o0 = Y * s1.y + X;  // X even: the pairs are 8-byte aligned
            const float2 w0 = __ldg(reinterpret_cast<const float2 *>(d.w + o0));
            const float2 w1 = __ldg(reinterpret_cast<const float2 *>(d.w + o0 + s1.y));
            if (w0.x == 0.f && w0.y == 0.f && w1.x == 0.f && w1.y == 0.f) continue;  // contributes exactly nothing
            wt[0][0] = w0.x; wt[0][1] = w0.y; wt[1][0] = w1.x; wt[1][1] = w1.y;
            const uint2 a = __ldg(reinterpret_cast<const uint2 *>(d.q + o0));
            const uint2 b = __ldg(reinterpret_cast<const uint2 *>(d.q + o0 + s1.y));
            const unsigned p[2][2] = {{a.x, a.y}, {b.x, b.y}};
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    g_rb[dy][dx] = word_rb(p[dy][dx]);
                    g_g[dy][dx] = word_g(p[dy][dx]);
                }
        } else {
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    wt[dy][dx] = 0.f;
                    g_rb[dy][dx] = g_g[dy][dx] = 0u;
                    if (!in[dy][dx]) continue;
                    const int o = (Y + dy) * s1.y + X + dx;
                    wt[dy][dx] = d.w[o];
                    const unsigned v = __ldg(d.q + o);
                    g_rb[dy][dx] = word_rb(v);
                    g_g[dy][dx] = word_g(v);
                }
        }
        // Laplacian = level - pyrUp(next level); both are bytes, the difference fits a signed 16-bit lane (and the
        // reference's saturation to int16 can never act)
        unsigned lap_rb[2][2];
        int lap_g[2][2];
        if (LV != 2) {
            const Nbr q = neighbours(X >> 1, Y >> 1, r.z >> 1, r.w >> 1, s1.w);
            unsigned u_rb[2][2], u_g[2][2];
            up_quad_lanes(d.uq, q, u_rb, u_g);
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    lap_rb[dy][dx] = __vsub2(g_rb[dy][dx], u_rb[dy][dx]);
                    lap_g[dy][dx] = (int)g_g[dy][dx] - (int)u_g[dy][dx];
                }
        } else {
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    lap_rb[dy][dx] = g_rb[dy][dx];
                    lap_g[dy][dx] = (int)g_g[dy][dx];
                }
        }
        // all four weights exactly 1 (the interior of a full-weight image): (short)trunc(L * 1.0f) == L
        const bool unit = LV != 2 && wt[0][0] == 1.f && wt[0][1] == 1.f && wt[1][0] == 1.f && wt[1][1] == 1.f;
        if (unit) {
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    acc_rb[dy][dx] = __vadd2(acc_rb[dy][dx], lap_rb[dy][dx]);
                    acc_g[dy][dx] += lap_g[dy][dx];
                }
        } else {
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    const int tr = trunc16(fmul((float)lane_lo(lap_rb[dy][dx]), wt[dy][dx]));
                    const int tb = trunc16(fmul((float)lane_hi(lap_rb[dy][dx]), wt[dy][dx]));
                    acc_rb[dy][dx] = __vadd2(acc_rb[dy][dx], lanes(tr, tb));
                    acc_g[dy][dx] += trunc16(fmul((float)lap_g[dy][dx], wt[dy][dx]));
                }
        }
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) wsum[dy][dx] = fadd(wsum[dy][dx], wt[dy][dx]);
    }

    if (A.partial) {
        // hand the partial sums of this rank's items to the rank that owns the region
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                if (!pv[dy][dx]) continue;
                const int o = (y + dy - A.ry0) * A.slab_pitch + (x + dx - A.rx0);
                A.slab_acc[o] = (int16_t)lane_lo(acc_rb[dy][dx]);
                A.slab_acc[A.slab_plane + o] = (int16_t)acc_g[dy][dx];
                A.slab_acc[2 * A.slab_plane + o] = (int16_t)lane_hi(acc_rb[dy][dx]);
                A.slab_w[o] = wsum[dy][dx];
            }
        return;
    }

    // blend step + collapse: v = sat16(pyrUp(C_{l+1}) + (short)trunc(acc / (wsum + eps)))
    int acc[2][2][3];  // the three accumulators of each pixel as sign-extended shorts
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            acc[dy][dx][0] = lane_lo(acc_rb[dy][dx]);
            acc[dy][dx][1] = (int)(short)acc_g[dy][dx];
            acc[dy][dx][2] = lane_hi(acc_rb[dy][dx]);
        }
    int v[2][2][3];
    float den[2][2];
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) den[dy][dx] = fadd(wsum[dy][dx], SB_WEIGHT_EPS);
    // n = (short)trunc(a / den) without a division where the weight sum is exactly 1 or exactly 0 (one full-weight
    // image, or nothing): den = fl(1 + 1e-5) = 1 + 84 ulp, so for an integer 0 < |a| <= 32768 the quotient lies
    // strictly between |a| - 1 and |a| (a * 1e-5 is far above the float spacing and below 1) and truncates to
    // a - sign(a); with weight sum 0 the accumulator is 0 as well and the same formula gives 0.
    const bool unit = (wsum[0][0] == 1.f || wsum[0][0] == 0.f) && (wsum[0][1] == 1.f || wsum[0][1] == 0.f) &&
                      (wsum[1][0] == 1.f || wsum[1][0] == 0.f) && (wsum[1][1] == 1.f || wsum[1][1] == 0.f);
    // weight sum exactly 2 (two full-weight images, the bulk of an overlap): den = fl(2 + 1e-5) = 2 + 42 ulp; for even
    // |a| = 2k the quotient is k (1 - 5e-6), strictly inside (k-1, k); for odd |a| = 2k+1 it lies inside (k, k+1/2):
    // either way it truncates to (|a| - 1) / 2 rounded toward zero, with the sign of a.
    const bool two = wsum[0][0] == 2.f && wsum[0][1] == 2.f && wsum[1][0] == 2.f && wsum[1][1] == 2.f;
    int nrm[2][2][3];
    if (unit) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    const int a = (int)(short)acc[dy][dx][c];
                    nrm[dy][dx][c] = a - (a > 0) + (a < 0);
                }
    } else if (two) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    const int a = (int)(short)acc[dy][dx][c];
                    nrm[dy][dx][c] = (a - ((a >> 31) | 1)) / 2;  // a == 0: -1 / 2 == 0
                }
    } else {
        float rr[2][2];
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) rr[dy][dx] = rcp_refined(den[dy][dx]);
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) nrm[dy][dx][c] = norm16(acc[dy][dx][c], den[dy][dx], rr[dy][dx]);
    }
    if (LV != 2) {
        const Nbr q = neighbours(x >> 1, y >> 1, A.up.w_px, A.up.h_px, A.up.pitch);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            int u[2][2];
            up_quad(A.up.c + c * A.up.plane, q, u);
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) v[dy][dx][c] = sat_s16(u[dy][dx] + nrm[dy][dx][c]);
        }
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) v[dy][dx][c] = nrm[dy][dx][c];
    }
    if (LV == 1) {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
            const int o = (y + dy) * A.cur.pitch + x;
#pragma unroll
            for (int c = 0; c < 3; ++c)
                *reinterpret_cast<unsigned *>(A.cur.c + c * A.cur.plane + o) = ((unsigned)v[dy][0][c] & 0xffffu) | ((unsigned)v[dy][1][c] << 16);
        }
        return;
    }
    if (LV == 2) {  // the launcher never uses this kernel for a 0-band blend, so the top level is never level 0
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                if (!pv[dy][dx]) continue;
                const int o = (y + dy) * A.cur.pitch + x + dx;
#pragma unroll
                for (int c = 0; c < 3; ++c) A.cur.c[c * A.cur.plane + o] = (int16_t)v[dy][dx][c];
            }
        return;
    }
    // level 0: mask, zero outside it, crop to the roi / the rank's strip, |v| saturated to uint8 (convertScaleAbs)
    const PanoOut &out = A.out;
    // the usual case (launch-uniform test): image + mask, even pitches and origin, buffers below 4 GB -- 32-bit offsets
    // and 2-byte stores; a quad whose two columns are both stored takes it
    const bool plain = out.rgb && out.mask && !out.s16 && ((out.rgb_pitch | out.mask_pitch | A.out_x0) & 1) == 0 &&
                       out.rgb_pitch * out.h < (1ll << 32);
    if (plain && x >= A.out_lo && x + 1 < A.out_hi) {
        const unsigned xo = (unsigned)(x - A.out_x0);
        unsigned o_rgb = (unsigned)y * (unsigned)out.rgb_pitch + 3u * xo, o_m = (unsigned)y * (unsigned)out.mask_pitch + xo;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
            if (y + dy < out.h) {
                const bool on0 = wsum[dy][0] > SB_WEIGHT_EPS, on1 = wsum[dy][1] > SB_WEIGHT_EPS;
                unsigned b[6];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    b[c] = on0 ? (unsigned)min(abs(v[dy][0][c]), 255) : 0u;
                    b[3 + c] = on1 ? (unsigned)min(abs(v[dy][1][c]), 255) : 0u;
                }
                unsigned short *p2 = reinterpret_cast<unsigned short *>(out.rgb + o_rgb);
                p2[0] = (unsigned short)(b[0] | (b[1] << 8));
                p2[1] = (unsigned short)(b[2] | (b[3] << 8));
                p2[2] = (unsigned short)(b[4] | (b[5] << 8));
                *reinterpret_cast<unsigned short *>(out.mask + o_m) = (unsigned short)((on0 ? 255u : 0u) | (on1 ? 0xff00u : 0u));
            }
            o_rgb += (unsigned)out.rgb_pitch;
            o_m += (unsigned)out.mask_pitch;
        }
        return;
    }
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
        if (y + dy >= out.h) continue;
        const bool s0 = x >= A.out_lo && x < A.out_hi, s1 = x + 1 >= A.out_lo && x + 1 < A.out_hi;  // column is stored?
        const bool on0 = wsum[dy][0] > SB_WEIGHT_EPS, on1 = wsum[dy][1] > SB_WEIGHT_EPS;
        const int xo = x - A.out_x0;  // column inside the output buffer
        if (out.rgb) {
            unsigned b[6];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                b[c] = on0 ? (unsigned)min(abs(v[dy][0][c]), 255) : 0u;
                b[3 + c] = on1 ? (unsigned)min(abs(v[dy][1][c]), 255) : 0u;
            }
            uint8_t *p = out.rgb + (long long)(y + dy) * out.rgb_pitch + 3 * xo;
            if (s0 && s1 && ((out.rgb_pitch | xo) & 1) == 0) {  // 2-byte aligned
                unsigned short *p2 = reinterpret_cast<unsigned short *>(p);
                p2[0] = (unsigned short)(b[0] | (b[1] << 8));
                p2[1] = (unsigned short)(b[2] | (b[3] << 8));
                p2[2] = (unsigned short)(b[4] | (b[5] << 8));
            } else {
                if (s0) { p[0] = (uint8_t)b[0]; p[1] = (uint8_t)b[1]; p[2] = (uint8_t)b[2]; }
                if (s1) { p[3] = (uint8_t)b[3]; p[4] = (uint8_t)b[4]; p[5] = (uint8_t)b[5]; }
            }
        }
        if (out.mask) {
            uint8_t *m = out.mask + (long long)(y + dy) * out.mask_pitch + xo;
            if (s0 && s1 && ((out.mask_pitch | xo) & 1) == 0) {
                *reinterpret_cast<unsigned short *>(m) = (unsigned short)((on0 ? 255u : 0u) | (on1 ? 0xff00u : 0u));
            } else {
                if (s0) m[0] = on0 ? 255 : 0;
                if (s1) m[1] = on1 ? 255 : 0;
            }
        }
        if (out.s16) {
            int16_t *d = out.s16 + (long long)(y + dy) * out.s16_pitch + 3 * xo;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                if (s0) d[c] = (int16_t)(on0 ? v[dy][0][c] : 0);
                if (s1) d[3 + c] = (int16_t)(on1 ? v[dy][1][c] : 0);
            }
        }
    }
}

}  // namespace

int launch_collapse(const CollapseArgs &A, int l, int nb, cudaStream_t s)
{
    const int rc = A.tile ? launch_collapse_tile(A, l, nb, s) : SB_ERR_STATE;
    if (rc != SB_ERR_STATE) return rc;
    if (A.rw <= 0 || A.rh <= 0) return SB_OK;
    if (A.n > SB_MAX_ITEMS) {
        set_error("collapse: %d items exceed SB_MAX_ITEMS=%d", A.n, SB_MAX_ITEMS);
        return SB_ERR_INVALID;
    }
    dim3 block(CF_BX, CF_BY), grid(div_up(A.rw, 2 * CF_BX), div_up(A.rh, 2 * CF_BY));
    if (l == nb)
        launch_pdl(k_collapse_fast<2>, grid, block, 0, s, A);
    else if (l == 0)
        launch_pdl(k_collapse_fast<0>, grid, block, 0, s, A);
    else
        launch_pdl(k_collapse_fast<1>, grid, block, 0, s, A);
    return launch_check("k_collapse_fast");
}

}  // namespace sb
