// sb_comm.cpp -- NCCL plumbing for the multi-GPU path (one process per GPU).  NCCL is resolved with
// dlopen at first use so that single-GPU users do not need it installed.
#include <dlfcn.h>

#include <cstring>

#include "sb_internal.h"

namespace {
struct ncclUniqueIdRaw { char internal[128]; };
typedef void *ncclComm_t;
typedef int (*fn_get_unique_id)(ncclUniqueIdRaw *);
typedef int (*fn_comm_init_rank)(ncclComm_t *, int, ncclUniqueIdRaw, int);
typedef int (*fn_comm_destroy)(ncclComm_t);
typedef const char *(*fn_get_error_string)(int);

void *g_nccl = nullptr;
fn_get_unique_id p_get_unique_id = nullptr;
fn_comm_init_rank p_comm_init_rank = nullptr;
fn_comm_destroy p_comm_destroy = nullptr;
fn_get_error_string p_err = nullptr;
ncclComm_t g_comm = nullptr;
int g_rank = 0, g_world = 1;

int load_nccl()
{
    if (g_nccl) return SB_OK;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *n : names) {
        g_nccl = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_nccl) break;
    }
    if (!g_nccl) {
        sb::set_error("NCCL not found: %s", dlerror());
        return SB_ERR_COMM;
    }
    p_get_unique_id = (fn_get_unique_id)dlsym(g_nccl, "ncclGetUniqueId");
    p_comm_init_rank = (fn_comm_init_rank)dlsym(g_nccl, "ncclCommInitRank");
    p_comm_destroy = (fn_comm_destroy)dlsym(g_nccl, "ncclCommDestroy");
    p_err = (fn_get_error_string)dlsym(g_nccl, "ncclGetErrorString");
    if (!p_get_unique_id || !p_comm_init_rank || !p_comm_destroy) {
        sb::set_error("NCCL library lacks required symbols");
        return SB_ERR_COMM;
    }
    return SB_OK;
}
int nccl_fail(int rc, const char *what)
{
    sb::set_error("NCCL error %d (%s) in %s", rc, p_err ? p_err(rc) : "?", what);
    return SB_ERR_COMM;
}
}  // namespace

namespace {
typedef int (*fn_send)(const void *, size_t, int, int, ncclComm_t, cudaStream_t);
typedef int (*fn_recv)(void *, size_t, int, int, ncclComm_t, cudaStream_t);
typedef int (*fn_group)(void);
fn_send p_send = nullptr;
fn_recv p_recv = nullptr;
fn_group p_group_start = nullptr, p_group_end = nullptr;
}  // namespace

namespace sb {
int comm_rank() { return g_rank; }
int comm_world() { return g_world; }
bool comm_ready() { return g_comm != nullptr; }

// One grouped point-to-point exchange on stream `s`: for every peer k, send sendb[k] bytes and receive recvb[k] bytes
// (either may be 0).  This is the overlap exchange of the sharded composite: only the slabs where footprints cross a
// strip boundary travel over NVLink, not pano-sized buffers (NCCL has no int16 reduction: the add happens in the
// consumer kernel, in rank order).
int comm_exchange(int n, const int *peers, void *const *sendp, const size_t *sendb, void *const *recvp, const size_t *recvb,
                  cudaStream_t s)
{
    if (!g_comm) {
        set_error("sharded composite: sb_comm_init has not been called");
        return SB_ERR_STATE;
    }
    if (!p_send) {
        p_send = (fn_send)dlsym(g_nccl, "ncclSend");
        p_recv = (fn_recv)dlsym(g_nccl, "ncclRecv");
        p_group_start = (fn_group)dlsym(g_nccl, "ncclGroupStart");
        p_group_end = (fn_group)dlsym(g_nccl, "ncclGroupEnd");
        if (!p_send || !p_recv || !p_group_start || !p_group_end) {
            set_error("NCCL library lacks ncclSend / ncclRecv / ncclGroupStart / ncclGroupEnd");
            return SB_ERR_COMM;
        }
    }
    const int ncclChar = 0;  // ncclInt8 / ncclChar
    int rc = p_group_start();
    if (rc) return nccl_fail(rc, "ncclGroupStart");
    for (int k = 0; k < n; ++k) {
        if (sendb[k]) {
            rc = p_send(sendp[k], sendb[k], ncclChar, peers[k], g_comm, s);
            if (rc) return nccl_fail(rc, "ncclSend");
        }
        if (recvb[k]) {
            rc = p_recv(recvp[k], recvb[k], ncclChar, peers[k], g_comm, s);
            if (rc) return nccl_fail(rc, "ncclRecv");
        }
    }
    rc = p_group_end();
    if (rc) return nccl_fail(rc, "ncclGroupEnd");
    return SB_OK;
}
}  // namespace sb

namespace sb {
// every rank contributes `bytes_per_rank` bytes (host), all ranks receive the concatenation in rank order (host)
int comm_allgather_bytes(const void *mine, void *all, size_t bytes_per_rank, cudaStream_t s)
{
    if (!g_comm) {
        set_error("comm_allgather_bytes: sb_comm_init has not been called");
        return SB_ERR_STATE;
    }
    typedef int (*fn_allgather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t);
    static fn_allgather p_allgather = (fn_allgather)dlsym(g_nccl, "ncclAllGather");
    if (!p_allgather) {
        set_error("NCCL library lacks ncclAllGather");
        return SB_ERR_COMM;
    }
    const size_t all_bytes = bytes_per_rank * (size_t)g_world;
    Staging st(s);
    uint8_t *d_in = st.tmp<uint8_t>(bytes_per_rank), *d_out = st.tmp<uint8_t>(all_bytes);
    st.copy(d_in, bytes_per_rank, mine, bytes_per_rank, bytes_per_rank, 1, cudaMemcpyHostToDevice);
    st.run([&] {
        const int nrc = p_allgather(d_in, d_out, bytes_per_rank, 0 /* ncclChar */, g_comm, s);
        return nrc ? nccl_fail(nrc, "ncclAllGather") : SB_OK;
    });
    st.down(all, all_bytes, d_out, all_bytes, all_bytes, 1);
    return st.finish();
}
}  // namespace sb

extern "C" {

int sb_comm_unique_id(uint8_t id[SB_COMM_ID_BYTES])
{
    SB_TRY(load_nccl());
    ncclUniqueIdRaw raw;
    int rc = p_get_unique_id(&raw);
    if (rc) return nccl_fail(rc, "ncclGetUniqueId");
    std::memcpy(id, raw.internal, SB_COMM_ID_BYTES);
    return SB_OK;
}

int sb_comm_init(const uint8_t id[SB_COMM_ID_BYTES], int rank, int world)
{
    SB_TRY(sb::ensure_device());
    SB_TRY(load_nccl());
    if (g_comm) {
        sb::set_error("sb_comm_init: communicator already initialised");
        return SB_ERR_STATE;
    }
    ncclUniqueIdRaw raw;
    std::memcpy(raw.internal, id, SB_COMM_ID_BYTES);
    int rc = p_comm_init_rank(&g_comm, world, raw, rank);
    if (rc) return nccl_fail(rc, "ncclCommInitRank");
    g_rank = rank;
    g_world = world;
    return SB_OK;
}

int sb_comm_destroy(void)
{
    if (g_comm && p_comm_destroy) p_comm_destroy(g_comm);
    g_comm = nullptr;
    g_rank = 0;
    g_world = 1;
    return SB_OK;
}

}  // extern "C"
