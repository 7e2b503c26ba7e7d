// sb_seam.cu -- SeamFinder.resize on the device (stitching/seam_finder.py:38-43): the LOW-resolution seam mask is
// dilated (3x3), resized to the FINAL-resolution warped size and ANDed with the warped mask; the result is the blend
// mask Blender.feed gets (stitcher.py:223-225, 254).
//
// Arithmetic (restated and pinned in oracle/stitch_oracle.c): cv.dilate(.., None) = 3x3 maximum ignoring pixels outside
// the image; the reference's positional arguments select cv.resize's default INTER_LINEAR, which for uint8 is OpenCV's
// 11-bit fixed-point bilinear: per-axis taps (index pair, weights summing to 2048) built on the HOST in the reference's
// float / double order (sb_geometry.cpp: resize_linear_taps), horizontal sums in int, vertical
// ((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16), then (+2) >> 2; an exact 2x reduction is the 2x2 box average.
#include "sb_device.cuh"
#include "sb_launch.h"

namespace sb {

namespace {

__global__ void k_dilate3x3(const uint8_t *__restrict__ src, int pitch, int w, int h, uint8_t *__restrict__ dst)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    int m = 0;
    for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
            const int yy = y + dy, xx = x + dx;
            if ((unsigned)yy < (unsigned)h && (unsigned)xx < (unsigned)w) m = max(m, (int)src[yy * pitch + xx]);
        }
    dst[y * w + x] = (uint8_t)m;
}

// taps: [i0 | i1 | c0 | c1] per axis, n_dst entries each
__global__ void k_resize_linear_and(const uint8_t *__restrict__ src, int sw, const int *__restrict__ tx, const int *__restrict__ ty,
                                    const uint8_t *__restrict__ mask, long long mask_pitch, uint8_t *__restrict__ dst,
                                    long long dst_pitch, int w, int h, int half)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    int v;
    if (half) {  // exact 2x reduction: cv::resize reroutes INTER_LINEAR to the 2x2 box filter
        const uint8_t *p = src + (2 * y) * sw + 2 * x;
        v = (p[0] + p[1] + p[sw] + p[sw + 1] + 2) >> 2;
    } else {
        const int x0 = tx[x], x1 = tx[w + x], a0 = tx[2 * w + x], a1 = tx[3 * w + x];
        const int y0 = ty[y], y1 = ty[h + y], b0 = ty[2 * h + y], b1 = ty[3 * h + y];
        const uint8_t *r0 = src + y0 * sw, *r1 = src + y1 * sw;
        const int h0 = r0[x0] * a0 + r0[x1] * a1, h1 = r1[x0] * a0 + r1[x1] * a1;  // scale 2048
        v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
        v = sat_u8(v);
    }
    if (mask) v &= mask[y * mask_pitch + x];
    dst[y * dst_pitch + x] = (uint8_t)v;
}

// cv.resize(uint8, cn channels, INTER_LINEAR_EXACT) (Images.resize_img_by_scaler, stitching/images.py:120-123): OpenCV's
// bit-exact 8.8 / 16.16 fixed-point bilinear (resize_exact_value); taps [i0 | i1 | c1] per axis from the host
// (resize_exact_taps)
__global__ void k_resize_exact(const uint8_t *__restrict__ src, long long spitch, int cn, const int *__restrict__ tx,
                               const int *__restrict__ ty, uint8_t *__restrict__ dst, long long dpitch, int w, int h)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const unsigned cx1 = (unsigned)tx[2 * w + x], cy1 = (unsigned)ty[2 * h + y];
    const uint8_t *r0 = src + ty[y] * spitch, *r1 = src + ty[h + y] * spitch;
    const int x0 = tx[x] * cn, x1 = tx[w + x] * cn;
    for (int c = 0; c < cn; ++c)
        dst[y * dpitch + (long long)x * cn + c] = (uint8_t)resize_exact_value(r0[x0 + c], r0[x1 + c], r1[x0 + c], r1[x1 + c], cx1, cy1);
}

}  // namespace

int launch_resize_exact(const uint8_t *src, long long spitch, int cn, const int *tx, const int *ty, uint8_t *dst, long long dpitch, int w,
                        int h, cudaStream_t s)
{
    launch(k_resize_exact, dim3(div_up(w, 32), div_up(h, 8)), dim3(32, 8), 0, s, src, spitch, cn, tx, ty, dst, dpitch, w, h);
    return launch_check("k_resize_exact");
}

// dst (w x h, device) = resize(dilate3x3(seam)) [& mask]; seam (sw x sh, device, pitch sw), scratch >= sw*sh bytes,
// tx / ty: device tap tables of the two axes (resize_linear_taps), ignored for the exact 2x reduction
int launch_seam_resize(const uint8_t *seam, int sw, int sh, uint8_t *scratch, const int *tx, const int *ty, const uint8_t *mask,
                       long long mask_pitch, uint8_t *dst, long long dst_pitch, int w, int h, cudaStream_t s)
{
    dim3 block(32, 8);
    launch(k_dilate3x3, dim3(div_up(sw, 32), div_up(sh, 8)), block, 0, s, seam, sw, sw, sh, scratch);
    SB_TRY(launch_check("k_dilate3x3"));
    const int half = sw == 2 * w && sh == 2 * h;
    launch(k_resize_linear_and, dim3(div_up(w, 32), div_up(h, 8)), block, 0, s, (const uint8_t *)scratch, sw, tx, ty, mask, mask_pitch, dst,
           dst_pitch, w, h, half);
    return launch_check("k_resize_linear_and");
}

}  // namespace sb
