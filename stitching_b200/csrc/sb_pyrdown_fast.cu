// sb_pyrdown_fast.cu -- instruction-lean pyrDown of one Gaussian/weight level for all fed images.
//
// Same arithmetic as k_pyrdown_gather (sb_pyramid.cu; reference chain stitching/blender.py:41 ->
// MultiBandBlender::feed -> copyMakeBorder + pyrDown(int16x3) + pyrDown(float32)).
//
// One warp walks down a strip of destination columns.  Lane k owns destination column x = strip + k - 1 and the
// source pair (2x, 2x+1); it gets the other three taps of the horizontal [1 4 6 4 1] from lanes k-1 and k+1 with
// warp shuffles.  Lanes 0 and 31 are HALO lanes: they own the virtual columns just outside the strip, load their
// pair like everybody else (through the same border index maps, so a virtual column beyond the level's edge holds
// exactly the reflected samples its neighbour needs) and store nothing -- 30 output columns per warp and not a
// single conditional load.  The five horizontally filtered rows live in registers as a sliding window (a
// destination row consumes two new source rows), so every source pixel is fetched once (plus a 3-row warm-up per
// chunk and the two halo pairs per row).  The two source rows of the NEXT destination row are requested before the
// current one is computed (software prefetch).  No shared memory, no atomics.
//   level 0 (packed RGBM bytes): red/blue and green run as two 16-bit lanes of one 32-bit word through both
//     filter passes (5x5 weights sum to 256, 256*255+128 < 2^16, so a lane never carries into its neighbour);
//     each lane converts its own two mask bytes to float (2^23 mantissa trick, exact, keeps the XU pipe free) and
//     the weights travel by shuffle as well;
//   levels >= 1 (lane pairs r|b<<16, g per pixel + float32 weights): the own pair is one 16-byte load and the colours
//     run through the same two-lane arithmetic; every level is written as lane pairs (one 8-byte store per pixel).
// The float summation orders (position dependent, sb_pyramid.cuh) are per-lane constants.
//
// BIN (level 0, every mask byte of the batch is 0 or 255 -- the warped validity masks of a compositor without blend
// masks): the weights w = mask * fl(1/255) are exactly 0 or 1, so every partial sum of the float pyrDown is a small
// integer and its value does not depend on the summation order: the level-1 weight is V / 256 with V = the integer
// 5x5 filter of the mask BITS.  The mask byte already rides through both integer passes in the spare 16-bit lane next
// to green (V_m = 255 V <= 65280), so the float path -- half of the kernel's instructions in the profile of the generic
// version -- disappears: V = (257 V_m + 65535) >> 16, one conversion, one exact multiply.
// The levels built from such weights stay exact for two more steps: level-1 weights are V / 2^8 (V <= 2^8), level-2
// weights V / 2^16, and every partial sum of the next pyrDown is an integer multiple of that unit not above 2^24 -- inside
// the float's 24-bit significand -- so for l = 1, 2 BIN means "any summation order": the kernel evaluates one instead of
// both.  From level 3 on the sums need up to 2^28 units and the reference's position-dependent orders matter again.
#include "sb_launch.h"
#include "sb_pyramid.cuh"

namespace sb {

namespace {

constexpr int WK_WARPS = 4;  // warps per block: consecutive row chunks of the same strip
constexpr int WK_COLS = 30;  // destination columns per warp (lanes 1..30; lanes 0 and 31 are halo lanes)
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float byte3_to_float(unsigned p)
{
    // bytes [p.byte3, 0, 0, 0x4B] = the float 2^23 + m; subtracting 2^23 is exact
    return fadd(__uint_as_float(__byte_perm(p, 0x4B000000u, 0x7443)), -8388608.f);
}

struct Raw0 { unsigned p2, p3; };                 // own pair of packed pixels (mask byte cleared outside the image)
struct H0 { unsigned rb, gm; float w; };
struct Raw1 { uint2 p2, p3; float2 wp; };         // own pair of lane-pair pixels + weights
struct H1 { unsigned rb, g; float w; };

// NEAR: every row index the walk produces is at most one reflection away from its range (the launcher checks the
// geometry of all images of the batch): the border rules are two selects instead of an integer modulo per row.
template <bool L0, bool NEAR, bool BIN>
__global__ void __launch_bounds__(32 * WK_WARPS, (L0 && BIN) ? 12 : 10) k_pyrdown_walk(const PyrDesc *__restrict__ descs, int rows_per_warp)
{
    const PyrDesc &D = descs[blockIdx.z];
    const int4 da = __ldg(reinterpret_cast<const int4 *>(&D.sw));  // sw, sh, dpitch, dplane
    const int sw = da.x, sh = da.y, dw = sw >> 1, dh = sh >> 1;
    const int lane = threadIdx.x;
    const int strip = blockIdx.x * WK_COLS;
    const int y_begin = (blockIdx.y * WK_WARPS + threadIdx.y) * rows_per_warp;
    grid_dependency_sync();                    // (the descriptors above are written once, at plan time)
    if (strip >= dw || y_begin >= dh) return;  // warp-uniform
    const int y_end = min(y_begin + rows_per_warp, dh);
    const int x = strip + lane - 1;            // -1 .. dw: virtual columns at both ends
    const bool stores = lane >= 1 && lane <= WK_COLS && x < dw;

    // every descriptor field goes to registers once (the stores below could alias it otherwise)
    const int4 db = __ldg(reinterpret_cast<const int4 *>(&D.ih));          // ih, left, top, spitch
    const int2 dc = __ldg(reinterpret_cast<const int2 *>(&D.rgbm_pitch));  // rgbm_pitch, iw
    const uint32_t *__restrict__ rgbm = D.rgbm;
    const uint2 *__restrict__ sq = D.sq;
    const float *__restrict__ swt = D.swt;
    uint2 *__restrict__ dq = D.dq;
    float *__restrict__ dwt = D.dwt;
    const int ih = db.x, left = db.y, top = db.z, spitch = db.w, rgbm_pitch = dc.x, iw = dc.y;

    // own pair (2x, 2x+1) through the level's border rule; at level 0 additionally into the fed image.
    // For x in [0, dw) the pair is (2x, 2x+1) itself; the virtual columns x = -1 and x >= dw reflect.
    const int xc = min(x, dw);  // columns beyond dw are never used by a storing lane: keep the indices tame
    int c2 = reflect101(2 * xc, sw), c3 = reflect101(2 * xc + 1, sw);
    const bool pair_adjacent = c3 == c2 + 1;
    unsigned keep2 = 0xffffffffu, keep3 = 0xffffffffu;  // level 0: mask byte survives only inside the fed image
    if (L0) {
        c2 -= left;
        c3 -= left;
        if ((unsigned)c2 >= (unsigned)iw) keep2 = 0x00ffffffu;
        if ((unsigned)c3 >= (unsigned)iw) keep3 = 0x00ffffffu;
        c2 = reflect(c2, iw);
        c3 = reflect(c3, iw);
    }
    const bool h_simd = x >= 1 && x < pyrdown_hs_end(sw);
    const bool v_simd = x < (dw / 4) * 4;

    auto fetch0 = [&](int src_row) -> Raw0 {
        const int iy = (NEAR ? reflect101_once(src_row, sh) : reflect101(src_row, sh)) - top;
        const unsigned rowkeep = (unsigned)iy < (unsigned)ih ? 0xffffffffu : 0x00ffffffu;
        const uint32_t *row = rgbm + (NEAR ? reflect_once(iy, ih) : reflect(iy, ih)) * rgbm_pitch;
        Raw0 r;
        r.p2 = __ldg(row + c2) & keep2 & rowkeep;  // outside the fed image the weight is 0: 0 * (1/255) == 0 exactly
        r.p3 = __ldg(row + c3) & keep3 & rowkeep;
        return r;
    };
    auto hpass0 = [&](const Raw0 &r) -> H0 {
        const unsigned p0 = __shfl_up_sync(FULL, r.p2, 1), p1 = __shfl_up_sync(FULL, r.p3, 1);
        const unsigned p4 = __shfl_down_sync(FULL, r.p2, 1);
        const unsigned M = 0x00ff00ffu;
        H0 h;
        h.rb = (p0 & M) + (p4 & M) + 4u * ((p1 & M) + (r.p3 & M)) + 6u * (r.p2 & M);
        h.gm = __byte_perm(p0, 0u, 0x4341) + __byte_perm(p4, 0u, 0x4341) +
               4u * (__byte_perm(p1, 0u, 0x4341) + __byte_perm(r.p3, 0u, 0x4341)) + 6u * __byte_perm(r.p2, 0u, 0x4341);
        if (BIN) {
            h.w = 0.f;  // the weight is read off the mask lane of gm after the vertical pass
        } else {
            const float w2 = fmul(byte3_to_float(r.p2), SB_INV255), w3 = fmul(byte3_to_float(r.p3), SB_INV255);
            const float w0 = __shfl_up_sync(FULL, w2, 1), w1 = __shfl_up_sync(FULL, w3, 1), w4 = __shfl_down_sync(FULL, w2, 1);
            h.w = tap5_h(w0, w1, w2, w3, w4, h_simd);
        }
        return h;
    };
    auto fetch1 = [&](int src_row) -> Raw1 {
        const int ro = (NEAR ? reflect101_once(src_row, sh) : reflect101(src_row, sh)) * spitch;
        Raw1 r;
        if (pair_adjacent) {  // (2x, 2x+1): one 16-byte / 8-byte load (true for every real column)
            const uint4 v = __ldg(reinterpret_cast<const uint4 *>(sq + ro + c2));
            r.p2 = make_uint2(v.x, v.y);
            r.p3 = make_uint2(v.z, v.w);
            r.wp = __ldg(reinterpret_cast<const float2 *>(swt + ro + c2));
        } else {              // a reflected virtual column
            r.p2 = __ldg(sq + ro + c2);
            r.p3 = __ldg(sq + ro + c3);
            r.wp.x = __ldg(swt + ro + c2);
            r.wp.y = __ldg(swt + ro + c3);
        }
        return r;
    };
    auto hpass1 = [&](const Raw1 &r) -> H1 {
        H1 h;
        {
            const unsigned p0 = __shfl_up_sync(FULL, r.p2.x, 1), p1 = __shfl_up_sync(FULL, r.p3.x, 1), p4 = __shfl_down_sync(FULL, r.p2.x, 1);
            h.rb = p0 + p4 + 4u * (p1 + r.p3.x) + 6u * r.p2.x;
        }
        {
            const unsigned p0 = __shfl_up_sync(FULL, r.p2.y, 1), p1 = __shfl_up_sync(FULL, r.p3.y, 1), p4 = __shfl_down_sync(FULL, r.p2.y, 1);
            h.g = p0 + p4 + 4u * (p1 + r.p3.y) + 6u * r.p2.y;
        }
        const float w0 = __shfl_up_sync(FULL, r.wp.x, 1), w1 = __shfl_up_sync(FULL, r.wp.y, 1);
        const float w4 = __shfl_down_sync(FULL, r.wp.x, 1);
        h.w = tap5_h(w0, w1, r.wp.x, r.wp.y, w4, BIN ? true : h_simd);
        return h;
    };

    const int dpitch = da.z;
    if (L0) {
        H0 h0 = hpass0(fetch0(2 * y_begin - 2)), h1 = hpass0(fetch0(2 * y_begin - 1)), h2 = hpass0(fetch0(2 * y_begin));
        Raw0 ra = fetch0(2 * y_begin + 1), rb = fetch0(2 * y_begin + 2);
        for (int y = y_begin; y < y_end; ++y) {
            Raw0 na = ra, nb = rb;
            if (y + 1 < y_end) {  // request the next two source rows before touching the current ones
                na = fetch0(2 * y + 3);
                nb = fetch0(2 * y + 4);
            }
            const H0 h3 = hpass0(ra), h4 = hpass0(rb);
            if (stores) {
                const unsigned vrb = h0.rb + h4.rb + 4u * (h1.rb + h3.rb) + 6u * h2.rb + 0x00800080u;
                const unsigned vgm = h0.gm + h4.gm + 4u * (h1.gm + h3.gm) + 6u * h2.gm + 0x00800080u;
                const int o = y * dpitch + x;
                dq[o] = make_uint2((vrb >> 8) & 0x00ff00ffu, (vgm >> 8) & 0xffu);
                if (BIN) {
                    const unsigned vm = (vgm >> 16) - 128u;                    // 255 * (filtered mask bits), <= 65280
                    dwt[o] = fmul((float)((vm * 257u + 65535u) >> 16), 0.00390625f);
                } else {
                    dwt[o] = tap5_v(h0.w, h1.w, h2.w, h3.w, h4.w, v_simd);
                }
            }
            h0 = h2;
            h1 = h3;
            h2 = h4;
            ra = na;
            rb = nb;
        }
    } else {
        H1 h0 = hpass1(fetch1(2 * y_begin - 2)), h1 = hpass1(fetch1(2 * y_begin - 1)), h2 = hpass1(fetch1(2 * y_begin));
        Raw1 ra = fetch1(2 * y_begin + 1), rb = fetch1(2 * y_begin + 2);
        for (int y = y_begin; y < y_end; ++y) {
            Raw1 na = ra, nb = rb;
            if (y + 1 < y_end) {
                na = fetch1(2 * y + 3);
                nb = fetch1(2 * y + 4);
            }
            const H1 h3 = hpass1(ra), h4 = hpass1(rb);
            if (stores) {
                const unsigned vrb = h0.rb + h4.rb + 4u * (h1.rb + h3.rb) + 6u * h2.rb + 0x00800080u;
                const unsigned vg = h0.g + h4.g + 4u * (h1.g + h3.g) + 6u * h2.g + 128u;
                const int o = y * dpitch + x;
                dq[o] = make_uint2((vrb >> 8) & 0x00ff00ffu, vg >> 8);
                dwt[o] = tap5_v(h0.w, h1.w, h2.w, h3.w, h4.w, BIN ? true : v_simd);
            }
            h0 = h2;
            h1 = h3;
            h2 = h4;
            ra = na;
            rb = nb;
        }
    }
}

}  // namespace

int launch_pyrdown_fast(const PyrDesc *pyr, const FeedImage *imgs_host, int count, int l, int max_w, int max_h, cudaStream_t s, bool binary_masks)
{
    // rows per warp: long chunks amortise the 3-row warm-up, but the small levels need more warps in flight
    long long strips = 0;
    for (int i = 0; i < count; ++i) strips += (long long)div_up((imgs_host[i].pw >> (l + 1)), WK_COLS) * ((imgs_host[i].ph >> (l + 1)));
    int rows = 32;
    while (rows > 4 && strips / rows < 16384) rows >>= 1;
    dim3 block(32, WK_WARPS), grid(div_up(max_w, WK_COLS), div_up(div_up(max_h, rows), WK_WARPS), count);
    // single-reflection border rules: source rows run from -2 to sh+1 (needs sh >= 4); at level 0 the padded rect may
    // not reach further beyond the fed image than the image is high
    bool near = true;
    for (int i = 0; i < count; ++i) {
        const FeedImage &im = imgs_host[i];
        near = near && (im.ph >> l) >= 4;
        if (l == 0) near = near && im.top <= im.h && im.ph - im.top - im.h <= im.h;
    }
    if (l == 0 && binary_masks && near)
        launch_lanes(k_pyrdown_walk<true, true, true>, grid, block, 0, s, pyr, rows);
    else if (l == 0 && binary_masks)
        launch_lanes(k_pyrdown_walk<true, false, true>, grid, block, 0, s, pyr, rows);
    else if (l == 0 && near)
        launch_lanes(k_pyrdown_walk<true, true, false>, grid, block, 0, s, pyr, rows);
    else if (l == 0)
        launch_lanes(k_pyrdown_walk<true, false, false>, grid, block, 0, s, pyr, rows);
    else if (l <= 2 && binary_masks && near)  // weights still exact in any order (see the header)
        launch_lanes(k_pyrdown_walk<false, true, true>, grid, block, 0, s, pyr, rows);
    else if (near)
        launch_lanes(k_pyrdown_walk<false, true, false>, grid, block, 0, s, pyr, rows);
    else
        launch_lanes(k_pyrdown_walk<false, false, false>, grid, block, 0, s, pyr, rows);
    return launch_check("k_pyrdown_walk");
}

}  // namespace sb
