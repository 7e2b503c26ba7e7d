// sb_pyramid.cu -- Gaussian pyramid construction of the fed images (colours int16 x3, weights float32).
//
// Replaces the pyrDown chain of MultiBandBlender::feed (createLaplacePyr on the int16 image and the
// pyrDown loop over the weight map), reached from stitching/blender.py:41.  The padded copy of the image
// (copyMakeBorder) is never materialised: level 0 is read through index maps (sb_pyramid.cuh).
#include <algorithm>
#include <cstdlib>

#include "sb_launch.h"
#include "sb_gather.cuh"

namespace sb {

namespace {

constexpr int PD_BX = 32, PD_BY = 8;

// simple variant: one thread per destination pixel, 25 gathered taps
__global__ void __launch_bounds__(PD_BX *PD_BY) k_pyrdown_gather(const FeedImage *__restrict__ imgs, int first, int l)
{
    const FeedImage &im = imgs[first + blockIdx.z];
    const int dw = im.pw >> (l + 1), dh = im.ph >> (l + 1);  // destination level size
    const int x = blockIdx.x * PD_BX + threadIdx.x;
    const int y = blockIdx.y * PD_BY + threadIdx.y;
    if (x >= dw || y >= dh) return;

    pyrdown_pixel(im, l, x, y);
}


}  // namespace

int launch_pyrdown_fast(const PyrDesc *pyr, const FeedImage *imgs_host, int count, int l, int max_w, int max_h,
                        cudaStream_t s, bool binary_masks);  // sb_pyrdown_fast.cu

int launch_pyrdown(const FeedImage *imgs_dev, const FeedImage *imgs_host, const PyrDesc *pyr, int first, int count, int l,
                   cudaStream_t s, bool binary_masks)
{
    // max_w / max_h: largest DESTINATION level size among the images of the batch.  The fast kernel works on byte-fed
    // images (RGBM level 0, one colour word per pixel above); generic int16 feeds use the gather kernel
    int max_w = 0, max_h = 0;
    bool packed = true;
    for (int i = first; i < first + count; ++i) {
        max_w = std::max(max_w, imgs_host[i].pw >> (l + 1));
        max_h = std::max(max_h, imgs_host[i].ph >> (l + 1));
        packed = packed && imgs_host[i].rgbm != nullptr;
    }
    if (count <= 0 || max_w <= 0 || max_h <= 0) return SB_OK;
#ifdef SB_EMU
    // the emulation plays a warp's 32 lanes with 32 host threads: correct but slow, so the shuffle kernel runs there only
    // on request (tests/test_host_logic.py sets SB_EMU_LANES around a small case); otherwise the gather kernel
    if (!getenv("SB_EMU_LANES")) packed = false;
#endif
    if (!use_simple_kernels() && packed) return launch_pyrdown_fast(pyr + first, imgs_host + first, count, l, max_w, max_h, s, binary_masks);
    dim3 block(PD_BX, PD_BY), grid(div_up(max_w, PD_BX), div_up(max_h, PD_BY), count);
    launch(k_pyrdown_gather, grid, block, 0, s, imgs_dev, first, l);
    return launch_check("k_pyrdown_gather");
}

}  // namespace sb
