// sb_feather_fast.cu -- feather weights: w = min(L1 distance to the nearest zero mask pixel * sharpness, 1).
//
// Replaces createWeightMap of cv.detail_FeatherBlender (stitching/blender.py:34-36, :41):
// distanceTransform(mask, DIST_L1, 3) + multiply + threshold(TRUNC 1).  The exact city-block distance is separable:
// d(x,y) = min_y' ( r(x,y') + |y - y'| ) with r = distance along the row to the nearest zero of that row.
//   rows:    one warp per row; per 32-pixel chunk a ballot gives the zero positions.  The ballots of a whole row stay in
//            registers (lane c & 31 keeps the word of chunk c), two warp scans turn them into "nearest zero before /
//            after this chunk", and one store per chunk writes min(x - left zero, right zero - x): every mask byte is
//            loaded once, nothing is read back, no load waits for a carried value (k_dt_rows_bits; rows wider than
//            32 * 32 * DT_WORDS pixels take the two-sweep kernel k_dt_rows_warp).
//   columns: with slope-1 costs the min-plus sweeps are prefix minima: going down d(y) = y + min_{j<=y}(r(j) - j), going
//            up d(y) = -y + min_{j>=y}(r(j) + j).  A column is cut into SB_DT_CHUNKS row chunks with one thread each:
//            k_dt_cols_summary reduces every chunk to its two minima, k_dt_cols_apply combines the minima of the chunks
//            above / below into carries and walks its own chunk down and up -- the serial chain is h / 32 rows instead
//            of 2 h (the one-thread-per-column sweeps of k_dt_cols_batched were most of a 16 x 2000x1500 feather
//            blend where they were measured).  All images of the blend in one launch each.
// "No zero anywhere" stays at DT_INF and becomes weight 1, as with OpenCV (the image border is not a zero).
#include <cstdlib>

#include "sb_launch.h"
#include "sb_pyramid.cuh"

namespace sb {

namespace {

#define DT_INF (1 << 29)
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ unsigned mask_at(const FeedImage &im, int x, int y)
{
    if (im.rgbm) return __ldg(im.rgbm + (long long)y * im.rgbm_pitch + x) >> 24;
    return im.mask[(long long)y * im.mask_pitch + x];
}

__global__ void __launch_bounds__(256) k_dt_rows_warp(const FeedImage *__restrict__ imgs)
{
    grid_dependency_sync();
    const FeedImage &im = imgs[blockIdx.y];
    const int y = blockIdx.x * 8 + threadIdx.y, lane = threadIdx.x, w = im.w;
    if (y >= im.h) return;  // warp-uniform
    int *d = (int *)im.fw + (long long)y * w;
    int last = -(1 << 30);  // column of the nearest zero seen so far
    for (int b = 0; b < w; b += 32) {
        const int x = b + lane;
        const bool inb = x < w;
        const unsigned zeros = __ballot_sync(FULL, inb && mask_at(im, inb ? x : 0, y) == 0u);
        const unsigned le = zeros & (FULL >> (31 - lane));
        const int lz = le ? b + 31 - __clz(le) : last;
        if (inb) d[x] = min(x - lz, DT_INF);
        if (zeros) last = b + 31 - __clz(zeros);
    }
    int next = 1 << 30;
    for (int b = ((w - 1) / 32) * 32; b >= 0; b -= 32) {
        const int x = b + lane;
        const bool inb = x < w;
        const int dl = inb ? d[x] : DT_INF;
        const unsigned zeros = __ballot_sync(FULL, inb && dl == 0);
        const unsigned ge = zeros & (FULL << lane);
        const int nz = ge ? b + __ffs(ge) - 1 : next;
        if (inb) d[x] = min(dl, min(nz - x, DT_INF));
        if (zeros) next = b + __ffs(zeros) - 1;
    }
}

// ---- rows, one pass --------------------------------------------------------------------------------------------------
constexpr int DT_WORDS_MAX = 8;  // ballot words a lane keeps: rows up to 32 * 32 * 8 = 8192 pixels

template <int DT_WORDS>
__global__ void __launch_bounds__(256) k_dt_rows_bits(const FeedImage *__restrict__ imgs)
{
    grid_dependency_sync();
    const FeedImage &im = imgs[blockIdx.y];
    const int y = blockIdx.x * 8 + threadIdx.y, lane = threadIdx.x, w = im.w;
    if (y >= im.h) return;  // warp-uniform
    const int nchunks = (w + 31) >> 5;
    unsigned word[DT_WORDS];  // word[k]: zero positions of chunk 32 k + lane
#pragma unroll
    for (int k = 0; k < DT_WORDS; ++k) {
        word[k] = 0u;
        if (32 * k < nchunks) {  // warp-uniform
            // eight chunks at a time: all eight loads are in flight before the first ballot needs its value
            for (int c0 = 32 * k; c0 < min(32 * k + 32, nchunks); c0 += 8) {
                unsigned m[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int x = 32 * (c0 + j) + lane;
                    m[j] = x < w ? mask_at(im, x, y) : 1u;
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const unsigned zeros = __ballot_sync(FULL, m[j] == 0u);
                    if (lane == ((c0 + j) & 31)) word[k] = zeros;
                }
            }
        }
    }
    // column of the nearest zero in the chunks before / after each chunk: an exclusive max- / min-scan over the chunks
    int left[DT_WORDS], right[DT_WORDS];
    int carry = -(1 << 30);
#pragma unroll
    for (int k = 0; k < DT_WORDS; ++k) {
        left[k] = carry;
        if (32 * k < nchunks) {
            int v = word[k] ? 32 * (32 * k + lane) + 31 - __clz(word[k]) : -(1 << 30);  // last zero of the own chunk
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int o = (int)__shfl_up_sync(FULL, (unsigned)v, d);
                if (lane >= d) v = max(v, o);
            }
            int ex = (int)__shfl_up_sync(FULL, (unsigned)v, 1);  // inclusive -> exclusive
            if (lane == 0) ex = -(1 << 30);
            left[k] = max(ex, carry);
            carry = max(carry, (int)__shfl_sync(FULL, (unsigned)v, 31));
        }
    }
    carry = 1 << 30;
#pragma unroll
    for (int k = DT_WORDS - 1; k >= 0; --k) {
        right[k] = carry;
        if (32 * k < nchunks) {
            int v = word[k] ? 32 * (32 * k + lane) + __ffs(word[k]) - 1 : (1 << 30);  // first zero of the own chunk
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int o = (int)__shfl_down_sync(FULL, (unsigned)v, d);
                if (lane + d < 32) v = min(v, o);
            }
            int ex = (int)__shfl_down_sync(FULL, (unsigned)v, 1);
            if (lane == 31) ex = 1 << 30;
            right[k] = min(ex, carry);
            carry = min(carry, (int)__shfl_sync(FULL, (unsigned)v, 0));
        }
    }
    int *d = (int *)im.fw + (long long)y * w;
#pragma unroll
    for (int k = 0; k < DT_WORDS; ++k) {
        if (32 * k < nchunks) {
            for (int c = 32 * k; c < min(32 * k + 32, nchunks); ++c) {
                const int src = c & 31, x = 32 * c + lane;
                const unsigned zeros = __shfl_sync(FULL, word[k], src);
                const int lc = (int)__shfl_sync(FULL, (unsigned)left[k], src), rc = (int)__shfl_sync(FULL, (unsigned)right[k], src);
                const unsigned le = zeros & (FULL >> (31 - lane)), ge = zeros & (FULL << lane);
                const int lz = le ? 32 * c + 31 - __clz(le) : lc;
                const int nz = ge ? 32 * c + __ffs(ge) - 1 : rc;
                if (x < w) d[x] = min(min(x - lz, nz - x), DT_INF);
            }
        }
    }
}

// ---- columns, chunked prefix minima ------------------------------------------------------------------------------------
__device__ __forceinline__ void dt_chunk(int h, int ty, int *y0, int *y1)
{
    const int rows = (h + SB_DT_CHUNKS - 1) / SB_DT_CHUNKS;
    *y0 = min(ty * rows, h);
    *y1 = min(*y0 + rows, h);
}

__global__ void __launch_bounds__(256) k_dt_cols_summary(const FeedImage *__restrict__ imgs)
{
    const FeedImage &im = imgs[blockIdx.z];
    const int x = blockIdx.x * 32 + threadIdx.x, ty = blockIdx.y * 8 + threadIdx.y, w = im.w;
    if (x >= w) return;
    int y0, y1;
    dt_chunk(im.h, ty, &y0, &y1);
    const int *r = (const int *)im.fw + x;
    int dn = 1 << 30, up = 1 << 30;
#pragma unroll 8
    for (int y = y0; y < y1; ++y) {
        const int v = r[(long long)y * w];
        dn = min(dn, v - y);
        up = min(up, v + y);
    }
    im.dts[ty * w + x] = dn;
    im.dts[(SB_DT_CHUNKS + ty) * w + x] = up;
}

__global__ void __launch_bounds__(256) k_dt_cols_apply(const FeedImage *__restrict__ imgs, float sharpness)
{
    const FeedImage &im = imgs[blockIdx.z];
    const int x = blockIdx.x * 32 + threadIdx.x, ty = blockIdx.y * 8 + threadIdx.y, w = im.w;
    if (x >= w) return;
    int y0, y1;
    dt_chunk(im.h, ty, &y0, &y1);
    if (y0 >= y1) return;
    int run = 1 << 30;  // min over the chunks above of r(j) - j
    for (int t = 0; t < ty; ++t) run = min(run, im.dts[t * w + x]);
    int *d = (int *)im.fw + x;
    // eight rows at a time: the loads of a batch are independent of its stores (the compiler cannot know that rows do
    // not alias and would otherwise serialise load -> store -> load down the chunk)
    constexpr int B = 8;
    for (int yb = y0; yb < y1; yb += B) {
        int v[B];
#pragma unroll
        for (int k = 0; k < B; ++k) v[k] = yb + k < y1 ? d[(long long)(yb + k) * w] : (1 << 30);
#pragma unroll
        for (int k = 0; k < B; ++k) {
            run = min(run, v[k] - (yb + k));
            v[k] = run + yb + k;  // distance to the nearest zero at or above (may exceed DT_INF: "none")
        }
#pragma unroll
        for (int k = 0; k < B; ++k)
            if (yb + k < y1) d[(long long)(yb + k) * w] = v[k];
    }
    run = 1 << 30;      // min over the chunks below of r(j) + j
    for (int t = ty + 1; t < SB_DT_CHUNKS; ++t) run = min(run, im.dts[(SB_DT_CHUNKS + t) * w + x]);
    float *f = (float *)im.fw + x;
    for (int yb = y1 - 1; yb >= y0; yb -= B) {
        // inside the own chunk the downward distances stand in for r: d_down(j) + j - y >= the true distance through
        // row j and equals it for the zero's own row (derivation in DESIGN.md 3.3)
        int v[B];
#pragma unroll
        for (int k = 0; k < B; ++k) v[k] = yb - k >= y0 ? d[(long long)(yb - k) * w] : (1 << 30);
        float o[B];
#pragma unroll
        for (int k = 0; k < B; ++k) {
            const int y = yb - k;
            run = min(run, v[k] + y);
            const int dist_i = min(v[k], run - y);
            const float dist = dist_i >= DT_INF ? 3.402823466e+38f : (float)dist_i;
            o[k] = fminf(fmul(dist, sharpness), 1.f);
        }
#pragma unroll
        for (int k = 0; k < B; ++k)
            if (yb - k >= y0) f[(long long)(yb - k) * w] = o[k];
    }
}

__global__ void __launch_bounds__(128) k_dt_cols_batched(const FeedImage *__restrict__ imgs, float sharpness)
{
    const FeedImage &im = imgs[blockIdx.y];
    const int x = blockIdx.x * blockDim.x + threadIdx.x, w = im.w, h = im.h;
    if (x >= w) return;
    int *d = (int *)im.fw + x;
    int run = DT_INF;
#pragma unroll 8
    for (int y = 0; y < h; ++y) {
        run = min(d[(long long)y * w], min(run + 1, DT_INF));
        d[(long long)y * w] = run;
    }
    run = DT_INF;
    float *f = (float *)im.fw + x;
#pragma unroll 8
    for (int y = h - 1; y >= 0; --y) {
        run = min(d[(long long)y * w], min(run + 1, DT_INF));
        const float dist = run >= DT_INF ? 3.402823466e+38f : (float)run;
        f[(long long)y * w] = fminf(fmul(dist, sharpness), 1.f);
    }
}

}  // namespace

int launch_feather_weights_fast(const FeedImage *imgs_dev, const FeedImage *imgs_host, int n, float sharpness, cudaStream_t s)
{
    int mw = 0, mh = 0;
    for (int i = 0; i < n; ++i) {
        mw = mw > imgs_host[i].w ? mw : imgs_host[i].w;
        mh = mh > imgs_host[i].h ? mh : imgs_host[i].h;
    }
    if (n <= 0 || mw <= 0 || mh <= 0) return SB_OK;
    bool scratch = true;
    for (int i = 0; i < n; ++i) scratch = scratch && imgs_host[i].dts != nullptr;
    static const bool old_kernels = [] {
        const char *e = getenv("SB_DT");
        return e && e[0] == '0';  // SB_DT=0: the round-1 sweeps (A/B)
    }();
    if (mw <= 32 * 32 * 2 && !old_kernels)
        launch_lanes(k_dt_rows_bits<2>, dim3(div_up(mh, 8), n), dim3(32, 8), 0, s, imgs_dev);
    else if (mw <= 32 * 32 * DT_WORDS_MAX && !old_kernels)
        launch_lanes(k_dt_rows_bits<DT_WORDS_MAX>, dim3(div_up(mh, 8), n), dim3(32, 8), 0, s, imgs_dev);
    else
        launch_lanes(k_dt_rows_warp, dim3(div_up(mh, 8), n), dim3(32, 8), 0, s, imgs_dev);
    if (scratch && !old_kernels) {
        const dim3 grid(div_up(mw, 32), SB_DT_CHUNKS / 8, n), block(32, 8);
        launch(k_dt_cols_summary, grid, block, 0, s, imgs_dev);
        launch(k_dt_cols_apply, grid, block, 0, s, imgs_dev, sharpness);
    } else {
        launch(k_dt_cols_batched, dim3(div_up(mw, 128), n), dim3(128), 0, s, imgs_dev, sharpness);
    }
    return launch_check("k_dt_*");
}

}  // namespace sb
