// sb_util.cu -- small utility kernels (L2 flush for benchmarking hygiene).
#include "sb_device.cuh"
#include <algorithm>

#include "sb_launch.h"

namespace sb {
namespace {
__global__ void k_flush(uint4 *p, size_t n, unsigned v)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) p[i] = make_uint4(v, v, v, v);
}

__device__ __forceinline__ unsigned long long mix64(unsigned long long z)
{
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

// rcp_refined / fdiv_by (sb_device.cuh) against __fdiv_rn over the ranges their callers guarantee:
// mode 0 (warp kernel): b in [2^-60, 2^60], a = 0 or |a / b| in about [2^-40, 2^60], random signs and mantissas;
// mode 1 (collapse kernel): a an int16 value, b = w + 1e-5 with w a sum of up to 256 weights in [0, 1].
__global__ void k_selftest_division(unsigned long long n, unsigned long long seed, int mode, unsigned long long *bad)
{
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x, local = 0;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const unsigned long long h = mix64(seed + i), h2 = mix64(h);
        float a, b;
        if (mode == 0) {
            const int be = (int)(h % 121) - 60, qe = (int)((h >> 8) % 101) - 40;
            b = __uint_as_float(((unsigned)(be + 127) << 23) | ((unsigned)(h >> 20) & 0x7fffffu));
            a = __uint_as_float(((unsigned)(be + qe + 127) << 23) | ((unsigned)(h2 >> 20) & 0x7fffffu) | ((unsigned)(h2 & 1) << 31));
            if (b > 0x1p60f) b = 0x1p60f;
            if ((h2 >> 1) % 61 == 0) a = 0.f;
        } else {
            a = (float)((int)(h % 65536) - 32768);
            const unsigned k = (unsigned)(h2 % 5);
            float w = k == 0 ? 0.f : k == 1 ? 1.f : k == 2 ? 2.f : __uint_as_float(0x3f800000u | ((unsigned)(h2 >> 8) & 0x7fffffu)) - 1.f;
            if (k == 4) w = __fmul_rn(w, (float)((h2 >> 40) % 256 + 1));
            b = __fadd_rn(w, 1e-5f);
        }
        const float q = fdiv_by(a, b, rcp_refined(b)), ref = __fdiv_rn(a, b);
        local += (__float_as_uint(q) != __float_as_uint(ref)) && !(q == 0.f && ref == 0.f);
    }
    if (local) atomicAdd(bad, local);
}
}  // namespace

int launch_selftest_division(unsigned long long n, unsigned long long seed, int mode, unsigned long long *bad_dev, cudaStream_t s)
{
    launch(k_selftest_division, dim3(sm_count() * 8), dim3(256), 0, s, n, seed, mode, bad_dev);
    return launch_check("k_selftest_division");
}

#ifndef SB_EMU
// One warp polls up to 32 flags in this device's memory until each has reached `value` (flags only ever grow).  The
// sharded composite orders its ranks with this instead of cuStreamWaitValue32: an unsatisfied stream wait sends the
// channel back to the runlist and is re-examined a timeslice later, which slows the step down badly once steps are
// enqueued ahead; a polling warp sees the
// peer's write within a microsecond.
__global__ void k_wait_flags(const volatile unsigned *flags, unsigned mask, unsigned value)
{
    if ((mask >> threadIdx.x) & 1u) {
        while ((int)(flags[threadIdx.x] - value) < 0) __nanosleep(100);
    }
    __threadfence_system();  // the slabs written before the flag are visible to what follows in the stream
}
#endif

int launch_wait_flags(const unsigned *flags, unsigned mask, unsigned value, cudaStream_t s)
{
#ifndef SB_EMU
    if (!mask) return SB_OK;
    launch(k_wait_flags, dim3(1), dim3(32), 0, s, (const volatile unsigned *)flags, mask, value);
    return launch_check("k_wait_flags");
#else
    return SB_ERR_STATE;
#endif
}

// Timelapser frame (stitching/timelapser.py:40-52 -> cv::detail::Timelapser::process + getDst + convertScaleAbs): the
// canvas of the prepared roi, zero everywhere except ONE image pasted at (dx, dy) -- pixels that fall outside the canvas
// are dropped -- shown as min(|v|, 255).  One pass writes every canvas byte (no memset), four canvas bytes per thread
// where the row allows it.
__global__ void k_timelapse_frame(const uint8_t *__restrict__ src8, const int16_t *__restrict__ src16, long long spitch, int sw, int sh, int dx,
                                  int dy, uint8_t *__restrict__ dst, long long dpitch, int cw, int ch)
{
    const int y = blockIdx.y;
    const long long row_bytes = 3ll * cw;
    const int sy = y - dy;
    const bool row_in = (unsigned)sy < (unsigned)sh;
    uint8_t *drow = dst + (long long)y * dpitch;
    for (long long b = (long long)(blockIdx.x * blockDim.x + threadIdx.x); b < row_bytes; b += (long long)gridDim.x * blockDim.x) {
        unsigned v = 0u;
        if (row_in) {
            const int x = (int)(b / 3), c = (int)(b - 3ll * x), sx = x - dx;
            if ((unsigned)sx < (unsigned)sw) {
                if (src8) {
                    v = src8[(long long)sy * spitch + 3ll * sx + c];
                } else {
                    const int q = src16[(long long)sy * spitch + 3ll * sx + c];
                    const int a = q < 0 ? -q : q;  // |-32768| = 32768 saturates like every value above 255
                    v = a > 255 ? 255u : (unsigned)a;
                }
            }
        }
        drow[b] = (uint8_t)v;
    }
}

int launch_timelapse_frame(const uint8_t *src8, const int16_t *src16, long long spitch, int sw, int sh, int dx, int dy, uint8_t *dst,
                           long long dpitch, int cw, int ch, cudaStream_t s)
{
    if (cw <= 0 || ch <= 0) return SB_OK;
    const int bx = (int)std::min<long long>((3ll * cw + 255) / 256, 64);
    launch(k_timelapse_frame, dim3(bx, ch), dim3(256), 0, s, src8, src16, spitch, sw, sh, dx, dy, dst, dpitch, cw, ch);
    return launch_check("k_timelapse_frame");
}

// overwrite a buffer larger than L2 so that the next kernel starts from a cold cache
int launch_flush_l2(void *buf, size_t bytes, cudaStream_t s)
{
    static unsigned v = 0;
    launch(k_flush, dim3(sm_count() * 8), dim3(256), 0, s, (uint4 *)buf, bytes / sizeof(uint4), ++v);
    return launch_check("k_flush");
}
}  // namespace sb
