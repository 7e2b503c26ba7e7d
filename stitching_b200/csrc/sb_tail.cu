// sb_tail.cu -- the tail of the multiband pyramid in ONE launch: pyrDown of levels T .. nb-1 of every fed image, then
// accumulate + normalise + collapse of levels nb .. T of the panorama.
//
// From level 3 on a level is a few hundred thousand pixels: the round-1 launch list shows twelve short launches
// each for them (pyrDown l3-l6, collapse l7-l3) at under 10 % occupancy -- launch latency
// and the serial row walk of the tuned kernels, not work.  Here a persistent grid (two CTAs per SM) runs the phases
// back to back with a grid barrier in between, every phase as independent per-pixel gathers (sb_gather.cuh, the same
// functions as the simple kernels: bit-identical arithmetic, either level layout).  No location is read before the
// phase that writes it has passed the barrier and none is written twice, so the L1 caches cannot hold a stale line.
//
// The emulation build (tests/emu) has no concurrent CTAs to meet at a barrier: launch_tail reports SB_ERR_STATE there
// and the caller launches the per-level kernels.
#include "sb_gather.cuh"
#include "sb_launch.h"

namespace sb {

#ifndef SB_EMU
namespace {

constexpr int TAIL_THREADS = 256;

// sense-reversing grid barrier on two words in global memory ([0] arrivals, [1] generation); all CTAs are resident
// (the launcher sizes the grid from the occupancy calculator)
__device__ __forceinline__ void grid_barrier(unsigned *state, unsigned nblocks)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        volatile unsigned *gen = state + 1;
        const unsigned g = *gen;
        __threadfence();  // this CTA's stores of the phase are visible device-wide before it arrives
        if (atomicAdd(state, 1u) == nblocks - 1u) {
            *state = 0u;
            __threadfence();
            atomicAdd(state + 1, 1u);
        } else {
            while (*gen == g) __nanosleep(64);
        }
        __threadfence();
    }
    __syncthreads();
}

struct TailArgs {
    const FeedImage *imgs;
    const PanoLevel *pano;
    int first, count, n;  // pyramids of images [first, first + count); the collapse sees all n
    int T, nb;
    int wp, hp;           // padded pano size at level 0
    PanoOut out;          // used when T == 0
    unsigned *state;
};

__global__ void __launch_bounds__(TAIL_THREADS) k_pyramid_tail(const __grid_constant__ TailArgs A)
{
    __shared__ int cum[SB_MAX_IMAGES + 1];
    const unsigned nblocks = gridDim.x;
    const long long stride = (long long)nblocks * TAIL_THREADS;
    const long long t0 = (long long)blockIdx.x * TAIL_THREADS + threadIdx.x;
    for (int l = A.T; l < A.nb; ++l) {
        // destination pixels of all images as one index space: cum[i] = pixels of the images before image i
        if (threadIdx.x == 0) {
            int c = 0;
            for (int i = 0; i < A.count; ++i) {
                cum[i] = c;
                const FeedImage &im = A.imgs[A.first + i];
                c += (im.pw >> (l + 1)) * (im.ph >> (l + 1));
            }
            cum[A.count] = c;
        }
        __syncthreads();
        const int total = cum[A.count];
        int i = 0;
        for (long long t = t0; t < total; t += stride) {
            while (t >= cum[i + 1]) ++i;
            const FeedImage &im = A.imgs[A.first + i];
            const int dw = im.pw >> (l + 1), r = (int)t - cum[i];
            pyrdown_pixel(im, l, r % dw, r / dw);
        }
        grid_barrier(A.state, nblocks);
    }
    for (int l = A.nb; l >= A.T; --l) {
        const int lw = l == 0 ? A.out.w : A.wp >> l, lh = l == 0 ? A.out.h : A.hp >> l;
        const long long total = (long long)lw * lh;
        for (long long t = t0; t < total; t += stride) collapse_pixel(A.imgs, A.n, A.pano, l, A.nb, (int)(t % lw), (int)(t / lw), A.out);
        if (l > A.T) grid_barrier(A.state, nblocks);
    }
}

}  // namespace

int launch_tail(const FeedImage *imgs_dev, const PanoLevel *pano_dev, int first, int count, int n, int T, int nb, int wp, int hp, const PanoOut &out,
                unsigned *state, cudaStream_t s)
{
    static int blocks_per_sm = -1;
    if (blocks_per_sm < 0) {
        int b = 0;
        SB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_pyramid_tail, TAIL_THREADS, 0));
        blocks_per_sm = b;
    }
    if (blocks_per_sm < 1 || count > SB_MAX_IMAGES) return SB_ERR_STATE;
    TailArgs A;
    A.imgs = imgs_dev;
    A.pano = pano_dev;
    A.first = first;
    A.count = count;
    A.n = n;
    A.T = T;
    A.nb = nb;
    A.wp = wp;
    A.hp = hp;
    A.out = out;
    A.state = state;
    const int grid = sm_count() * (blocks_per_sm < 2 ? blocks_per_sm : 2);
    launch(k_pyramid_tail, dim3(grid), dim3(TAIL_THREADS), 0, s, A);
    return launch_check("k_pyramid_tail");
}
#else
int launch_tail(const FeedImage *, const PanoLevel *, int, int, int, int, int, int, int, const PanoOut &, unsigned *, cudaStream_t) { return SB_ERR_STATE; }
#endif

}  // namespace sb
