// sb_peer.cpp -- the slab exchange of the sharded composite as direct NVLink stores (no reference counterpart: the
// reference is single-process; this is SURVEY.md 8(e)).
//
// Round 1 moved the slabs with grouped ncclSend / ncclRecv on a communication stream: at 8 GPUs the exchange ran far
// below link rate and the collapse waited for it (VERDICT r1, item 8).  Here every rank keeps the slabs it RECEIVES
// in one cudaMalloc'ed arena, exports it with CUDA IPC, and maps its neighbours' arenas.  The partial-sum launches
// (k_collapse_fast with `partial` set) write their slabs into local send buffers and the copy engines move them into
// the owners' arenas (cudaMemcpyAsync on the mapped peer pointers: NVLink DMA at link rate, no SM, no NCCL kernel, on
// a second stream beside the pyramid kernels).  Storing the slabs from the kernels straight into the peers' arenas is
// available too (SB_PEER=direct) -- it lost where it was measured: the 2- and 4-byte scattered stores of that kernel
// cross NVLink as small partial writes.  The ranks order themselves with four flags per pair, written by
// stream memory operations (cuStreamWriteValue32: stream-ordered behind the copy, no host round trip) and awaited by a
// one-warp polling kernel (k_wait_flags, sb_util.cu) right before the kernel that reads the slab -- cuStreamWaitValue32
// was measured too and lost: enqueued ahead, the front end evaluates those waits in batches:
//   data[part][p]  in the RECEIVER's arena: rank p has finished writing part `part` (0: level 0, 1: the coarser
//                  levels) of step `value`;
//   consumed[p]    in the SENDER's arena: rank p has read the slabs of step `value` (the next step may overwrite them).
// NCCL stays the bootstrap (all-gather of the IPC handles) and the fallback (SB_PEER=0, or a failing connect()).
#include <cstring>

#include "sb_shard.h"

#ifndef SB_EMU
#include <cuda.h>
#endif

namespace sb {

namespace {
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
}

size_t ShardPlan::arena_layout(const BlendPlan &plan, int dst, std::vector<size_t> *off, size_t *flags) const
{
    size_t o = 0;
    if (off) off->assign(world, 0);
    for (int src = 0; src < world; ++src) {
        if (src == dst) continue;
        PeerSlab ps;
        slab_geometry(plan, src, dst, &ps);
        if (off) (*off)[src] = o;
        o = align_up(o + ps.bytes, 256);
    }
    if (flags) *flags = o;
    return o + align_up(sizeof(unsigned) * 3 * (size_t)world, 256);  // data[0][world], data[1][world], consumed[world]
}

#ifndef SB_EMU
namespace {
typedef CUresult (*MemOpFn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
MemOpFn p_write = nullptr, p_wait = nullptr;
bool load_memops()
{
    if (p_write && p_wait) return true;
    cudaDriverEntryPointQueryResult q;
    void *a = nullptr, *b = nullptr;
    if (cudaGetDriverEntryPoint("cuStreamWriteValue32", &a, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) a = nullptr;
    if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &b, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) b = nullptr;
    (void)cudaGetLastError();
    p_write = (MemOpFn)a;
    p_wait = (MemOpFn)b;
    return p_write && p_wait;
}
}  // namespace

int ShardPlan::connect(const BlendPlan &plan, cudaStream_t s)
{
    connected = false;
    const char *e = getenv("SB_PEER");
    direct_stores = e && !strcmp(e, "direct");
    if ((e && e[0] == '0') || !comm_ready() || comm_world() != world || comm_rank() != rank) return SB_OK;  // NCCL exchange
    if (!load_memops()) return SB_OK;
    // my arena: the slabs I receive (they replace the per-peer receive buffers) + the flags
    std::vector<size_t> off;
    arena_bytes = arena_layout(plan, rank, &off, &flags_off);
    SB_CUDA(cudaMalloc(&arena, arena_bytes));
    SB_CUDA(cudaMemsetAsync(arena, 0, arena_bytes, s));
    SB_CUDA(cudaStreamSynchronize(s));
    cudaIpcMemHandle_t mine;
    SB_CUDA(cudaIpcGetMemHandle(&mine, arena));
    std::vector<cudaIpcMemHandle_t> all(world);
    SB_TRY(comm_allgather_bytes(&mine, all.data(), sizeof mine, s));  // also a barrier: every arena is zeroed by now
    peer_arena.assign(world, nullptr);
    peer_slot.assign(world, 0);
    peer_flags_off.assign(world, 0);
    bool ok = true;
    for (int p = 0; p < world && ok; ++p) {
        if (p == rank || (!send[p].bytes && !recv[p].bytes)) continue;
        void *ptr = nullptr;
        if (cudaIpcOpenMemHandle(&ptr, all[p], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
            (void)cudaGetLastError();
            ok = false;
            break;
        }
        peer_arena[p] = (char *)ptr;
        std::vector<size_t> poff;
        size_t pflags = 0;
        arena_layout(plan, p, &poff, &pflags);
        peer_slot[p] = poff[rank];
        peer_flags_off[p] = pflags;
    }
    // all ranks take the same decision: one failing mapping sends everybody back to the NCCL exchange
    int mine_ok = ok ? 1 : 0;
    std::vector<int> oks(world, 0);
    SB_TRY(comm_allgather_bytes(&mine_ok, oks.data(), sizeof(int), s));
    for (int v : oks) ok = ok && v == 1;
    if (!ok) {
        for (auto &p : peer_arena)
            if (p) (void)cudaIpcCloseMemHandle(p);
        peer_arena.clear();
        (void)cudaFree(arena);
        arena = nullptr;
        return SB_OK;
    }
    // the receive slabs now live in the arena (the item lists are built from recv[p].buf afterwards, in allocate())
    recv_off = off;
    connected = true;
    step = 0;
    return SB_OK;
}

static int memop(MemOpFn fn, cudaStream_t s, void *addr, unsigned value, unsigned flags, const char *what)
{
    const CUresult r = fn((CUstream)s, (CUdeviceptr)(uintptr_t)addr, value, flags);
    if (r != CUDA_SUCCESS) {
        set_error("%s failed with %d", what, (int)r);
        return SB_ERR_CUDA;
    }
    return SB_OK;
}

int ShardPlan::push(cudaStream_t s, int part)
{
    for (int p = 0; p < world; ++p) {
        if (p == rank || !send[p].bytes || !peer_arena[p]) continue;
        const size_t s0 = part == 1 ? send[p].split : 0, s1 = part == 0 ? send[p].split : send[p].bytes;  // level 0 lies in front
        if (s1 <= s0) continue;
        SB_CUDA(cudaMemcpyAsync(peer_arena[p] + peer_slot[p] + s0, (const char *)send[p].buf + s0, s1 - s0, cudaMemcpyDeviceToDevice, s));
    }
    return SB_OK;
}

int ShardPlan::signal_data(cudaStream_t s, int part, unsigned value)
{
    for (int p = 0; p < world; ++p) {
        if (p == rank || !send[p].bytes || !peer_arena[p]) continue;
        unsigned *flags = (unsigned *)(peer_arena[p] + peer_flags_off[p]);
        SB_TRY(memop(p_write, s, flags + (size_t)part * world + rank, value, CU_STREAM_WRITE_VALUE_DEFAULT, "cuStreamWriteValue32"));
    }
    return SB_OK;
}
int ShardPlan::wait_data(cudaStream_t s, int part, unsigned value)
{
    if (world > 32) {
        set_error("sharded composite: the flag wait serves at most 32 ranks");
        return SB_ERR_INVALID;
    }
    unsigned *flags = (unsigned *)((char *)arena + flags_off) + (size_t)part * world;
    unsigned mask = 0;
    for (int p = 0; p < world; ++p)
        if (p != rank && recv[p].bytes) mask |= 1u << p;
    return launch_wait_flags(flags, mask, value, s);  // a polling warp (sb_util.cu), not cuStreamWaitValue32
}
int ShardPlan::signal_consumed(cudaStream_t s, unsigned value)
{
    for (int p = 0; p < world; ++p) {
        if (p == rank || !recv[p].bytes || !peer_arena[p]) continue;
        unsigned *flags = (unsigned *)(peer_arena[p] + peer_flags_off[p]);
        SB_TRY(memop(p_write, s, flags + (size_t)2 * world + rank, value, CU_STREAM_WRITE_VALUE_DEFAULT, "cuStreamWriteValue32"));
    }
    return SB_OK;
}
int ShardPlan::wait_consumed(cudaStream_t s, unsigned value)
{
    unsigned *flags = (unsigned *)((char *)arena + flags_off) + (size_t)2 * world;
    unsigned mask = 0;
    for (int p = 0; p < world; ++p)
        if (p != rank && send[p].bytes) mask |= 1u << p;
    return launch_wait_flags(flags, mask, value, s);
}
#else
int ShardPlan::connect(const BlendPlan &, cudaStream_t) { return SB_OK; }
int ShardPlan::push(cudaStream_t, int) { return SB_ERR_STATE; }
int ShardPlan::signal_data(cudaStream_t, int, unsigned) { return SB_ERR_STATE; }
int ShardPlan::wait_data(cudaStream_t, int, unsigned) { return SB_ERR_STATE; }
int ShardPlan::signal_consumed(cudaStream_t, unsigned) { return SB_ERR_STATE; }
int ShardPlan::wait_consumed(cudaStream_t, unsigned) { return SB_ERR_STATE; }
#endif

}  // namespace sb
