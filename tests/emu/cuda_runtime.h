// tests/emu/cuda_runtime.h -- TEST INFRASTRUCTURE ONLY.
// A CPU stand-in for the few CUDA runtime calls and device builtins libstitch_b200 uses, so that the product's
// host logic (plans, geometry, C ABI) and the arithmetic of its kernels can be exercised on a GPU-less box
// (pytest -m "not gpu"): synchronisation-free kernels run as serial loops over the grid (sb_emu_run), kernels whose
// lanes exchange values through warp shuffles run with 32 host threads as the lanes of a warp (sb_emu_run_lanes),
// kernels whose threads share memory and meet at block barriers run with one host thread per thread of a block
// (sb_emu_run_block).
// The product build never sees this header (it is only on the include path of tests/emu/Makefile, which
// defines SB_EMU), the product loader (stitching_b200/_lib.py) never loads the emu library, and nothing
// measured or shipped runs through it.
#pragma once
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 };
typedef struct emuStream_st *cudaStream_t;
typedef struct emuEvent_st *cudaEvent_t;
typedef int cudaMemPool_t;
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum { cudaStreamNonBlocking = 1 };
enum cudaMemPoolAttr { cudaMemPoolAttrReleaseThreshold = 4 };
struct cudaDeviceProp { char name[256]; int major, minor, multiProcessorCount; };
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(8) int2 { int x, y; };
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(8) float2 { float x, y; };
static inline uint4 make_uint4(unsigned a, unsigned b, unsigned c, unsigned d) { return uint4{a, b, c, d}; }
static inline int4 make_int4(int a, int b, int c, int d) { return int4{a, b, c, d}; }
static inline int2 make_int2(int a, int b) { return int2{a, b}; }
static inline uint2 make_uint2(unsigned a, unsigned b) { return uint2{a, b}; }
// lane-wise 16-bit add / subtract with wrap-around (VIADD.16x2)
static inline unsigned __vadd2(unsigned a, unsigned b) { return ((a + b) & 0xffffu) | (((a >> 16) + (b >> 16)) << 16); }
static inline unsigned __vsub2(unsigned a, unsigned b) { return ((a - b) & 0xffffu) | (((a >> 16) - (b >> 16)) << 16); }

// lane-wise signed 16-bit min / max of (a + b) and c (VIADDMNMX.S16x2), lane-wise signed min (VIMNMX.S16x2)
static inline unsigned emu_lanes2(int lo, int hi) { return ((unsigned)lo & 0xffffu) | ((unsigned)hi << 16); }
static inline int emu_lo16(unsigned v) { return (int)(short)(v & 0xffffu); }
static inline int emu_hi16(unsigned v) { return (int)(short)(v >> 16); }
static inline unsigned __viaddmin_s16x2(unsigned a, unsigned b, unsigned c)
{
    const int lo = (short)(emu_lo16(a) + emu_lo16(b)), hi = (short)(emu_hi16(a) + emu_hi16(b));
    return emu_lanes2(lo < emu_lo16(c) ? lo : emu_lo16(c), hi < emu_hi16(c) ? hi : emu_hi16(c));
}
static inline unsigned __viaddmax_s16x2(unsigned a, unsigned b, unsigned c)
{
    const int lo = (short)(emu_lo16(a) + emu_lo16(b)), hi = (short)(emu_hi16(a) + emu_hi16(b));
    return emu_lanes2(lo > emu_lo16(c) ? lo : emu_lo16(c), hi > emu_hi16(c) ? hi : emu_hi16(c));
}
static inline unsigned __vmins2(unsigned a, unsigned b)
{
    return emu_lanes2(emu_lo16(a) < emu_lo16(b) ? emu_lo16(a) : emu_lo16(b), emu_hi16(a) < emu_hi16(b) ? emu_hi16(a) : emu_hi16(b));
}

static inline const char *cudaGetErrorString(cudaError_t) { return "emu"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 8; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { std::memset(p, 0, sizeof *p); std::strcpy(p->name, "EMU (tests only)"); p->major = 9; p->multiProcessorCount = 132; return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = (cudaStream_t)std::malloc(1); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { std::free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceGetDefaultMemPool(cudaMemPool_t *p, int) { *p = 0; return cudaSuccess; }
static inline cudaError_t cudaMemPoolSetAttribute(cudaMemPool_t, cudaMemPoolAttr, void *) { return cudaSuccess; }
static inline cudaError_t cudaMallocAsync(void **p, size_t n, cudaStream_t) { *p = std::malloc(n); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaFreeAsync(void *p, cudaStream_t) { std::free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void **p, size_t n) { *p = std::malloc(n); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaFreeHost(void *p) { std::free(p); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t) { std::memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t) { std::memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t)
{
    for (size_t y = 0; y < h; ++y) std::memcpy((char *)d + y * dp, (const char *)s + y * sp, w);
    return cudaSuccess;
}
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = (cudaEvent_t)std::malloc(1); return cudaSuccess; }
enum { cudaEventDisableTiming = 2 };
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = (cudaEvent_t)std::malloc(1); return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { std::free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 1.f; return cudaSuccess; }

// ---- device builtins ------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __grid_constant__
struct emuIdx { unsigned x, y, z; };
extern thread_local emuIdx threadIdx, blockIdx, blockDim, gridDim;
template <typename T> static inline T __ldg(const T *p) { return *p; }
// built with -ffp-contract=off: each op rounds once, like the __f*_rn intrinsics
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
static inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) { const unsigned long long o = *p; *p += v; return o; }
// byte / bit shuffles of the fast warp kernel
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh)
{
    sh &= 31u;
    return sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
}
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned sel)
{
    const unsigned long long v = ((unsigned long long)b << 32) | a;
    unsigned r = 0;
    for (int i = 0; i < 4; ++i) r |= (unsigned)((v >> (8 * ((sel >> (4 * i)) & 7u))) & 0xffu) << (8 * i);
    return r;
}
static inline unsigned __dp2a_lo(unsigned a, unsigned b, unsigned c) { return c + (a & 0xffffu) * (b & 0xffu) + (a >> 16) * ((b >> 8) & 0xffu); }
static inline int __float2int_rn(float v) { return (int)nearbyintf(v); }
static inline int __float2int_rz(float v) { return (int)v; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }

// ---- kernels whose lanes talk to each other (warp shuffles) -----------------------------------------------------
// 32 host threads play the 32 lanes; every thread walks all warps of the grid in the same order and the lanes meet at
// each collective (their control flow around collectives is warp-uniform, as CUDA requires for the *_sync forms).
struct EmuWarpSync {
    std::mutex m;
    std::condition_variable cv;
    int waiting = 0;
    unsigned long long generation = 0;
    unsigned vals[32];
    void barrier()
    {
        std::unique_lock<std::mutex> lk(m);
        const unsigned long long g = generation;
        if (++waiting == 32) {
            waiting = 0;
            ++generation;
            cv.notify_all();
        } else {
            cv.wait(lk, [&] { return generation != g; });
        }
    }
    unsigned exchange(unsigned lane, unsigned v, int src)  // every lane publishes v and reads lane `src` (own value if out of range)
    {
        vals[lane] = v;
        barrier();
        const unsigned r = (src >= 0 && src < 32) ? vals[src] : v;
        barrier();
        return r;
    }
};
extern thread_local EmuWarpSync *emu_warp;
static inline unsigned __ballot_sync(unsigned, int pred)
{
    emu_warp->vals[threadIdx.x] = pred ? 1u : 0u;
    emu_warp->barrier();
    unsigned m = 0;
    for (int i = 0; i < 32; ++i) m |= emu_warp->vals[i] << i;
    emu_warp->barrier();
    return m;
}
static inline int __all_sync(unsigned m, int pred) { return __ballot_sync(m, pred) == 0xffffffffu; }
static inline int __clz(unsigned v) { return v ? __builtin_clz(v) : 32; }
static inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline unsigned __shfl_up_sync(unsigned, unsigned v, unsigned d) { return emu_warp->exchange(threadIdx.x, v, (int)threadIdx.x - (int)d); }
static inline unsigned __shfl_down_sync(unsigned, unsigned v, unsigned d) { return emu_warp->exchange(threadIdx.x, v, (int)threadIdx.x + (int)d); }
static inline unsigned __shfl_sync(unsigned, unsigned v, int src) { return emu_warp->exchange(threadIdx.x, v, src & 31); }
static inline float __shfl_up_sync(unsigned m, float v, unsigned d) { return __uint_as_float(__shfl_up_sync(m, __float_as_uint(v), d)); }
static inline float __shfl_down_sync(unsigned m, float v, unsigned d) { return __uint_as_float(__shfl_down_sync(m, __float_as_uint(v), d)); }

template <typename F>
static inline void sb_emu_run_lanes(dim3 grid, dim3 block, F &&body)
{
    if (block.x != 32) std::abort();  // a warp is one row of the block in these kernels
    EmuWarpSync sync;
    std::vector<std::thread> lanes;
    for (unsigned lane = 0; lane < 32; ++lane)
        lanes.emplace_back([&, lane]() {
            emu_warp = &sync;
            gridDim = emuIdx{grid.x, grid.y, grid.z};
            blockDim = emuIdx{block.x, block.y, block.z};
            for (unsigned bz = 0; bz < grid.z; ++bz)
                for (unsigned by = 0; by < grid.y; ++by)
                    for (unsigned bx = 0; bx < grid.x; ++bx) {
                        blockIdx = emuIdx{bx, by, bz};
                        for (unsigned tz = 0; tz < block.z; ++tz)
                            for (unsigned ty = 0; ty < block.y; ++ty) {
                                threadIdx = emuIdx{lane, ty, tz};
                                body();
                            }
                    }
        });
    for (auto &t : lanes) t.join();
}

// ---- kernels whose threads share memory and meet at block barriers (sb_collapse_tile.cu) --------------------------
// One host thread per thread of a block; every host thread walks all blocks of the grid in the same order with its
// threadIdx fixed, __syncthreads is a rendezvous of all of them, the dynamic shared memory is one buffer they all see,
// and the warps (rows of 32 threads) get their own rendezvous for ballots.  A barrier at the end of every block keeps a
// fast thread from writing the next block's shared memory while a slow one still reads this block's.
struct EmuBlockSync {
    std::mutex m;
    std::condition_variable cv;
    int n = 0, waiting = 0;
    unsigned long long generation = 0;
    void barrier()
    {
        std::unique_lock<std::mutex> lk(m);
        const unsigned long long g = generation;
        if (++waiting == n) {
            waiting = 0;
            ++generation;
            cv.notify_all();
        } else {
            cv.wait(lk, [&] { return generation != g; });
        }
    }
};
extern thread_local EmuBlockSync *emu_block;
extern thread_local unsigned char *emu_smem;
static inline void __syncthreads()
{
    if (!emu_block) std::abort();  // a block-cooperative kernel was launched through the serial runner
    emu_block->barrier();
}

template <typename F>
static inline void sb_emu_run_block(dim3 grid, dim3 block, size_t smem_bytes, F &&body)
{
    if (block.x != 32 || block.z != 1) std::abort();
    EmuBlockSync sync;
    sync.n = (int)(block.x * block.y);
    std::vector<EmuWarpSync> warps(block.y);
    std::vector<unsigned char> smem(smem_bytes + 64);
    unsigned char *smem_base = smem.data() + ((64 - ((uintptr_t)smem.data() & 63)) & 63);
    std::vector<std::thread> threads;
    for (unsigned ty = 0; ty < block.y; ++ty)
        for (unsigned tx = 0; tx < block.x; ++tx)
            threads.emplace_back([&, tx, ty]() {
                emu_block = &sync;
                emu_warp = &warps[ty];
                emu_smem = smem_base;
                gridDim = emuIdx{grid.x, grid.y, grid.z};
                blockDim = emuIdx{block.x, block.y, block.z};
                threadIdx = emuIdx{tx, ty, 0};
                for (unsigned bz = 0; bz < grid.z; ++bz)
                    for (unsigned by = 0; by < grid.y; ++by)
                        for (unsigned bx = 0; bx < grid.x; ++bx) {
                            blockIdx = emuIdx{bx, by, bz};
                            body();
                            sync.barrier();
                        }
                emu_block = nullptr;
            });
    for (auto &t : threads) t.join();
}

template <typename F>
static inline void sb_emu_run(dim3 grid, dim3 block, F &&body)
{
    gridDim = emuIdx{grid.x, grid.y, grid.z};
    blockDim = emuIdx{block.x, block.y, block.z};
    for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
            for (unsigned bx = 0; bx < grid.x; ++bx) {
                blockIdx = emuIdx{bx, by, bz};
                for (unsigned tz = 0; tz < block.z; ++tz)
                    for (unsigned ty = 0; ty < block.y; ++ty)
                        for (unsigned tx = 0; tx < block.x; ++tx) {
                            threadIdx = emuIdx{tx, ty, tz};
                            body();
                        }
            }
}
