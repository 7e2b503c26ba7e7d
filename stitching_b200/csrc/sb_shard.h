// sb_shard.h -- one panorama composited by several GPUs (one process per GPU): image blocks per rank, pano column
// strips per rank, exchange of the per-band partial sums where footprints cross a strip boundary.
#pragma once
#include <vector>

#include "sb_plan.h"

namespace sb {

struct SlabLevel {
    int x0, y0, w, h;       // rectangle at this level, pano level coordinates (w == 0: nothing at this level)
    int pitch, plane;       // elements
    size_t acc_off, w_off;  // byte offsets inside the slab buffer
};
struct PeerSlab {
    SlabLevel lv[SB_MAX_BANDS + 1];
    size_t bytes = 0;       // 0: no exchange with this peer in this direction
    size_t split = 0;       // the level-0 part is [0, split), the coarser levels [split, bytes) (feather: split == bytes)
    void *buf = nullptr;    // device
    // byte range [*b, *e) of exchange part `part` (ShardPlan::parts)
    void part_range(int part, size_t *b, size_t *e) const
    {
        *b = part == 0 ? 0 : split;
        *e = part == 0 ? split : bytes;
    }
};

class ShardPlan {
public:
    int rank = 0, world = 1;
    int first = 0, count = 0;        // this rank's image block [first, first + count)
    bool feather = false;            // the feather blender (single level), else multiband
    std::vector<int> bounds;         // strip boundaries in padded-pano columns, world + 1 entries, multiples of 2^nb
                                     // (feather: in roi columns or rows, see `axis`)
    bool reversed = false;           // feather: the blocks follow each other against the axis (rank 0 owns the LAST strip)
    int axis = 0;                    // 0: column strips (multiband always); 1: row strips (feather, image blocks stacked vertically)
    std::vector<PeerSlab> send, recv;  // indexed by peer rank
    ColDesc *items_dev[SB_MAX_BANDS + 1] = {};
    TileDesc *tile_items_dev[SB_MAX_BANDS + 1] = {};  // the same lists for the tile kernels (null: images do not qualify)
    int n_items[SB_MAX_BANDS + 1] = {};
    // Direct exchange over NVLink (sb_peer.cpp): every rank's receive slabs live in ONE cudaMalloc'ed arena that its
    // neighbours map with CUDA IPC; copy-engine copies (or, with direct_stores, the partial-sum kernels themselves) put
    // the send slabs into the owners' arenas, and the ranks order themselves with flags written and awaited by stream
    // memory operations.  Not connected: the NCCL exchange is used.
    void *arena = nullptr;                 // recv slabs of all peers (rank order) + the flags
    size_t arena_bytes = 0, flags_off = 0;
    std::vector<size_t> recv_off;          // slab from peer p inside MY arena
    std::vector<char *> peer_arena;        // peer p's arena mapped into this process
    std::vector<size_t> peer_slot;         // offset of MY slab inside peer p's arena
    std::vector<size_t> peer_flags_off;    // offset of peer p's flags inside its arena
    bool connected = false;
    bool direct_stores = false;            // connected, SB_PEER=direct and multiband: the kernels store into the peers' arenas
    unsigned step = 0;                     // sharded steps issued so far (the flag values)

    static void block_of(int n_images, int world, int r, int *first, int *count)
    {
        *first = (int)((long long)r * n_images / world);
        *count = (int)((long long)(r + 1) * n_images / world) - *first;
    }
    // geometry from the plan of ALL images (identical on every rank)
    int build(const BlendPlan &plan, int rank, int world);
    // slab buffers, per-level item lists (own images + the slabs this rank receives) and the communication stream, after
    // plan.allocate()
    int allocate(const BlendPlan &plan, cudaStream_t s);
    void release(cudaStream_t s);
    // output columns (axis 0) / rows (axis 1) of this rank: [lo, hi) in pano-roi coordinates (may be empty)
    void strip(const BlendPlan &plan, int *lo, int *hi) const;

    // A sharded step moves its slabs in exchange parts: part 0 is level 0, part 1 the levels 1..nb (multiband only; the
    // feather blender has one level and one part).  Each part, in order: the work on the own images it reads, partial_out,
    // send_part.  Then, coarsest part first: receive_part, finish.  Level 0 -- three quarters of the bytes -- needs only
    // the first pyrDown and is collapsed last, so its slabs travel while the rest of the pyramid, the coarse parts and
    // their collapse run.
    int parts() const { return feather ? 1 : 2; }
    // partial sums of the own images over every region of the part a neighbour needs -> its send slab
    // (k_collapse_fast with `partial`, or k_feather_region)
    int partial_out(const BlendPlan &plan, int part, cudaStream_t s);
    // sum slabs + own images in rank order, normalise, collapse the own strip over the part's levels; `out` is strip-local
    int finish(const BlendPlan &plan, const PanoOut &out, int part, cudaStream_t s);
    // The transport (sb_peer.cpp), called on the compute stream s: the NCCL exchange on the communication stream, pushes
    // into the owners' arenas by the copy engines there, or with direct stores only the flags.  guard() goes right before
    // part 0's partial sums, which overwrite what the last step sent: with pushes it waits for the last step's copies,
    // with direct stores for the owners' "consumed" flags.  consumed() goes after the last finish: this rank has read the
    // slabs of this step.
    int guard(cudaStream_t s);
    int send_part(int part, cudaStream_t s);
    int receive_part(int part, cudaStream_t s);
    int consumed(cudaStream_t s);
    // direct exchange: layout of rank `dst`'s arena (same on every rank), IPC connection, flags
    size_t arena_layout(const BlendPlan &plan, int dst, std::vector<size_t> *off, size_t *flags) const;
    int connect(const BlendPlan &plan, cudaStream_t s);            // collective over the NCCL communicator

private:
    void slab_geometry(const BlendPlan &plan, int src, int dst, PeerSlab *ps) const;
    void feather_slab_geometry(const BlendPlan &plan, int src, int dst, PeerSlab *ps) const;
    int multiband_bounds(const BlendPlan &plan);
    int feather_bounds(const BlendPlan &plan);
    int exchange(int part, cudaStream_t s);                        // grouped NCCL send/recv of the part of every slab
    int push(int part, cudaStream_t s);                            // copy-engine copies of the part into the owners' arenas
    int signal_data(cudaStream_t s, int part, unsigned value);     // this rank has written part `part` of step `value`
    int wait_data(cudaStream_t s, int part, unsigned value);
    int signal_consumed(cudaStream_t s, unsigned value);           // this rank has read the slabs of step `value`
    int wait_consumed(cudaStream_t s, unsigned value);             // ... before the next ones overwrite them
    cudaStream_t comm_ = nullptr;                                  // NCCL exchange / pushes
    cudaEvent_t e_part_[2] = {}, e_xchg_[2] = {};                  // partial sums of part k written / part k exchanged
                                                                   // (pushes: the last part's copies done)
    void *feather_items_ = nullptr;  // FeatherSlab records of the slabs this rank receives (device)
    int feather_before_ = 0, feather_after_ = 0;
    void *items_arena_ = nullptr;
    void *tile_items_arena_ = nullptr;
};

int comm_allgather_bytes(const void *mine, void *all, size_t bytes_per_rank, cudaStream_t s);  // host buffers
int comm_rank();
int comm_world();
int comm_exchange(int n, const int *peers, void *const *sendp, const size_t *sendb, void *const *recvp, const size_t *recvb,
                  cudaStream_t s);
bool comm_ready();

}  // namespace sb
