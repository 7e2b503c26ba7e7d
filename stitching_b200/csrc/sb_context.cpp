// sb_context.cpp -- process-wide state of libstitch_b200.so: device selection, error text, launch
// counter, stream-ordered allocation.  One process drives one GPU (sb_init).
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <string>

#include "sb_internal.h"

namespace sb {

namespace {
thread_local char g_err[512] = "";
std::atomic<unsigned long long> g_launches{0};
std::mutex g_mu;
int g_device = -1;
int g_sm = 0;
cudaStream_t g_stream = nullptr;
cudaDeviceProp g_prop;
}  // namespace

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char *what, const char *file, int line)
{
    set_error("CUDA error %d (%s) at %s:%d in `%s`", (int)e, cudaGetErrorString(e), file, line, what);
    return e == cudaErrorMemoryAllocation ? SB_ERR_NOMEM : SB_ERR_CUDA;
}

void count_launch(unsigned n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
void adjust_launch_count(long long delta) { g_launches.fetch_add((unsigned long long)delta, std::memory_order_relaxed); }
int sm_count() { return g_sm; }
cudaStream_t default_stream() { return g_stream; }

static int init_locked(int ordinal)
{
    if (g_device == ordinal) return SB_OK;
    if (g_device >= 0) {
        set_error("sb_init: device %d already selected for this process (one process per GPU)", g_device);
        return SB_ERR_STATE;
    }
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        set_error("no CUDA device visible (%s); libstitch_b200 has no CPU fallback", e == cudaSuccess ? "count = 0" : cudaGetErrorString(e));
        (void)cudaGetLastError();
        return SB_ERR_NO_DEVICE;
    }
    if (ordinal < 0 || ordinal >= n) {
        set_error("sb_init: device ordinal %d out of range [0,%d)", ordinal, n);
        return SB_ERR_INVALID;
    }
    SB_CUDA(cudaSetDevice(ordinal));
    SB_CUDA(cudaGetDeviceProperties(&g_prop, ordinal));
#ifndef SB_EMU
    if (g_prop.major != 9 || g_prop.minor != 0) {
        set_error("device %d (%s) is sm_%d%d; libstitch_b200 is built for sm_90a only and has no fallback", ordinal, g_prop.name,
                  g_prop.major, g_prop.minor);
        return SB_ERR_NO_DEVICE;
    }
#endif
    SB_CUDA(cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking));
    cudaMemPool_t pool;
    SB_CUDA(cudaDeviceGetDefaultMemPool(&pool, ordinal));
    unsigned long long keep = ~0ull;  // keep freed blocks cached: prepare/feed/blend reuse them every stitch
    SB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    g_sm = g_prop.multiProcessorCount;
    g_device = ordinal;
    return SB_OK;
}

int ensure_device()
{
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_device >= 0) {
        // cudaSetDevice is per host thread: a caller on another thread than the one that initialised the library
        // would otherwise run on device 0 with streams of device g_device
        static thread_local int t_device = -1;
        if (t_device != g_device) {
            SB_CUDA(cudaSetDevice(g_device));
            t_device = g_device;
        }
        return SB_OK;
    }
    const char *env = getenv("SB_DEVICE");
    if (!env) env = getenv("LOCAL_RANK");
    return init_locked(env ? atoi(env) : 0);
}

int dev_alloc(void **p, size_t bytes, cudaStream_t s)
{
    *p = nullptr;
    if (bytes == 0) bytes = 16;
    SB_CUDA(cudaMallocAsync(p, bytes, s));
    return SB_OK;
}
void dev_free(void *p, cudaStream_t s)
{
    if (p) (void)cudaFreeAsync(p, s);
}

}  // namespace sb

extern "C" {

const char *sb_last_error(void) { return sb::g_err; }
const char *sb_version(void) { return "stitch_b200 0.1 (sm_90a)"; }

int sb_init(int device_ordinal)
{
    std::lock_guard<std::mutex> lk(sb::g_mu);
    return sb::init_locked(device_ordinal);
}

int sb_device_info(char *name, size_t name_len, int *sm_count, int *cc_major, int *cc_minor)
{
    SB_TRY(sb::ensure_device());
    if (name && name_len) snprintf(name, name_len, "%s", sb::g_prop.name);
    if (sm_count) *sm_count = sb::g_prop.multiProcessorCount;
    if (cc_major) *cc_major = sb::g_prop.major;
    if (cc_minor) *cc_minor = sb::g_prop.minor;
    return SB_OK;
}

unsigned long long sb_launch_count(void) { return sb::g_launches.load(); }

int sb_device_copy(void *dst, const void *src, size_t bytes)
{
    SB_TRY(sb::ensure_device());
    if (!bytes) return SB_OK;
    if (!dst || !src) {
        sb::set_error("sb_device_copy: null pointer");
        return SB_ERR_INVALID;
    }
    SB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, sb::g_stream));
    SB_CUDA(cudaStreamSynchronize(sb::g_stream));
    return SB_OK;
}

int sb_selftest_division(unsigned long long n, unsigned long long seed, int mode, unsigned long long *mismatches)
{
    SB_TRY(sb::ensure_device());
    if (!mismatches || mode < 0 || mode > 1) {
        sb::set_error("sb_selftest_division: bad arguments");
        return SB_ERR_INVALID;
    }
    unsigned long long *bad = nullptr;
    SB_TRY(sb::dev_alloc((void **)&bad, sizeof *bad, sb::g_stream));
    SB_CUDA(cudaMemsetAsync(bad, 0, sizeof *bad, sb::g_stream));
    int rc = sb::launch_selftest_division(n, seed, mode, bad, sb::g_stream);
    if (rc == SB_OK && cudaMemcpyAsync(mismatches, bad, sizeof *bad, cudaMemcpyDeviceToHost, sb::g_stream) != cudaSuccess) rc = SB_ERR_CUDA;
    if (rc == SB_OK && cudaStreamSynchronize(sb::g_stream) != cudaSuccess) rc = SB_ERR_CUDA;
    sb::dev_free(bad, sb::g_stream);
    return rc;
}

void *sb_host_alloc(size_t bytes)
{
    if (sb::ensure_device() != SB_OK) return nullptr;
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) {
        (void)cudaGetLastError();
        sb::set_error("cudaMallocHost(%zu) failed", bytes);
        return nullptr;
    }
    return p;
}
void sb_host_free(void *p)
{
    if (p) (void)cudaFreeHost(p);
}

}  // extern "C"

namespace sb {
bool pdl_enabled()
{
    static const bool on = [] {
        const char *e = getenv("SB_PDL");
        return !(e && e[0] == '0');
    }();
    return on;
}

bool use_simple_kernels()
{
    static const bool simple = [] {
        const char *e = getenv("SB_KERNELS");
        return e && std::string(e) == "simple";
    }();
    return simple;
}
}  // namespace sb
