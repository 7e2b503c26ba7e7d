// sb_collapse_tile.cu -- the per-level multiband kernel on shared-memory tiles (levels 0 .. nb-1).
//
// Same arithmetic as k_collapse_fast / k_collapse_gather (reference call chain stitching/blender.py:41,46 ->
// MultiBandBlender::feed / ::blend, SURVEY.md A.4): per pano pixel, in feed order over the images covering it,
//   L = G_l - pyrUp(G_{l+1});  acc += (short)trunc(L * w);  wsum += w;
// then n = (short)trunc(acc / (wsum + 1e-5)), C_l = sat16(pyrUp(C_{l+1}) + n), and at level 0 mask / |.| / uint8.
//
// What changed against k_collapse_fast is where the operands come from and how often they are touched.  The profile of
// k_collapse_fast shows 845 warp instructions per quad at level 0: 340 in the final pyrUp +
// store, ~190 per covering image, mostly address arithmetic, bounds tests and 9 + 27 scattered global taps per thread.
// Here a CTA owns a 64x16 tile (one thread per 2x2 quad) and stages every window the tile needs in shared memory with
// asynchronous 16-byte copies (cp.async / LDGSTS, zero fill outside the source, the next image's windows in flight
// while the current one is consumed): per covering image the 64x16 level-l pixels (level 0: packed RGBM; above: colour
// lane pairs + weights) and the 34x10 window of level l+1 that holds the 3x3 pyrUp neighbourhoods of all quads, plus
// the 34x10x3 window of the collapsed level C_{l+1}.  Elements outside a source arrive as zeros, which is exactly
// "weight 0": no rect tests and no predicated taps in the consumers, whose shared-memory loads sit at compile-time
// offsets.  The pyrUp is separable and neighbouring quads share two of their three coarse columns: every thread
// computes the vertical column sums of ONE coarse column into shared memory and reads its three columns back (3 + 3
// shared loads instead of 9 global ones per image, 9 + 6 instead of 27 for C_{l+1}).  The blend division, the
// collapse add and |.| / min run on two 16-bit lanes per word (VIADD.16x2, VIMNMX.S16x2) with exact integer forms
// for the weight sums 0, 1 and 2 that make up almost all of a panorama.
//
// (The first version staged the windows with the tensor copy engine, cp.async.bulk.tensor / UTMALDG.  The staging
// uses cp.async; sb_tma.cuh keeps the tensor-map wrappers.)
//
// Scope: byte-fed images, uint8 image + mask output, whole levels or a rank's strip of one (multi-GPU: the region may start
// anywhere even; the tile grid starts at the 64-column boundary at or left of it and quads left of the region are idle).
// Slabs of partial sums from other ranks (ColDesc kind 1) are items too: nothing is staged for them, every quad adds its
// four sums straight from global memory.  Producing partial sums, int16 output and the top level stay with
// k_collapse_fast (launch_collapse_tile says so by returning SB_ERR_STATE).  The emulation build (tests/emu)
// compiles the kernel as it is and runs it with one host thread per thread of a CTA (tests/emu: sb_emu_run_block; the
// asynchronous copies become plain copies) when SB_EMU_BLOCKS is set -- slow, hence on request only.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "sb_launch.h"
#include "sb_pyramid.cuh"

namespace sb {

namespace {

constexpr int TW = SB_TILE_W, TH = SB_TILE_H, QX = TW / 2, QY = TH / 2;  // 64 x 16 pixels, 32 x 8 quads
constexpr int UPW = SB_TILE_UPW, UPH = SB_TILE_UPH;
#define SB_WEIGHT_EPS 1e-5f

// Window geometry.  A staged row starts at a 16-byte boundary of its source row, so the logical window sits at a small
// column offset inside the staged one: the window of the collapsed level (origin = 32 k - 1 int16 elements) at +7; the
// windows of an image at offsets that depend on where its rect starts on the pano lattice (tile-uniform, run time):
// RGBM and weights at (tile_x - rect_x) & 3 elements, the 8-byte lane pairs of the coarser level at origin & 1.
constexpr int UPS = UPW + 2;                 // staged lane-pair window: 36 columns = 18 chunks, logical origin at +0 / +1 (run time)
constexpr int C1S = 48, C1O = 7;             // staged int16 window: 48 columns = 6 chunks
constexpr int RGS = TW + 4;                  // staged RGBM window: 68 pixels = 17 chunks

// the staged windows of one covering image
template <int LV>
struct ItemBuf;
template <>
struct alignas(16) ItemBuf<0> {
    uint32_t own[TH][RGS];  // packed RGBM, zero outside the image
    uint2 up[UPH][UPS];     // level-1 lane pairs around the tile
};
template <>
struct alignas(16) ItemBuf<1> {
    uint2 own[TH][TW];      // level-l lane pairs (rect origins are even: 16-byte rows)
    float w[TH][RGS];       // level-l weights, zero outside the padded rect
    uint2 up[UPH][UPS];
};

template <int LV>
struct Smem {
    ItemBuf<LV> item[2];                // the image being consumed and the next one in flight
    alignas(16) int16_t c1[3][UPH][C1S];
    alignas(16) uint4 cs[2][QY][UPW];   // column sums of the image in flight (double buffered); reused for C_{l+1}
    int list_n;
    unsigned short list[SB_MAX_ITEMS];
};

// 16-byte asynchronous copy global -> shared; `valid` false: nothing is read and the 16 bytes become zeros
#ifndef SB_EMU
__device__ __forceinline__ void cp_async16(void *dst, const void *src, bool valid)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
#else  // the emulation copies at once: the commit groups and waits have nothing left to do
__device__ __forceinline__ void cp_async16(void *dst, const void *src, bool valid)
{
    if (valid)
        std::memcpy(dst, src, 16);
    else
        std::memset(dst, 0, 16);
}
__device__ __forceinline__ void cp_async_commit() {}
template <int N>
__device__ __forceinline__ void cp_async_wait() {}
#endif

// One 16-byte chunk of a staged window: source row `row` (valid inside [0, rows_valid)), bytes [xb, xb + 16) of it
// (valid inside [0, row_bytes)); anything else arrives as zeros.  row_bytes is the valid width rounded UP to 16 bytes:
// the bytes between the valid width and row_bytes are the allocation's own zero-initialised row padding (BlendPlan /
// compositor).  Offsets fit 32 bits (the launcher checks the buffer sizes).
__device__ __forceinline__ void stage_chunk(void *dst, const void *base, unsigned pitch_b, int row, int rows_valid, int xb, int row_bytes)
{
    const bool ok = (unsigned)row < (unsigned)rows_valid && (unsigned)xb < (unsigned)row_bytes;
    const char *g = reinterpret_cast<const char *>(base) + (ok ? (unsigned)row * pitch_b + (unsigned)xb : 0u);
    cp_async16(dst, g, ok);
}

// pyrUp borders of a staged window (rows x cols elements, window origin (bx, by) in the source level of aw x ah
// elements): index -1 reads index 1 (reflect-101), index aw reads aw-1 (replicate); the copy engine delivered zeros
// there.  Only those two lines can be read by a quad inside the level.  Tile-uniform call (contains barriers).
// `t` points at logical column 0 of a staged window whose rows are STRIDE elements apart; COLS logical columns.
template <typename T, int ROWS, int COLS, int STRIDE>
__device__ __forceinline__ void fix_borders(T (*t)[STRIDE], int bx, int by, int aw, int ah, int tid)
{
    const int cl = -1 - bx, cr = aw - bx;  // window columns of index -1 and index aw
    if (tid < ROWS) {
        if (cl >= 0 && cl < COLS) t[tid][cl] = t[tid][min(cl + (aw > 1 ? 2 : 1), COLS - 1)];
        if (cr >= 1 && cr < COLS) t[tid][cr] = t[tid][cr - 1];
    }
    __syncthreads();
    const int rt = -1 - by, rb = ah - by;
    if (tid < COLS) {
        if (rt >= 0 && rt < ROWS) t[rt][tid] = t[min(rt + (ah > 1 ? 2 : 1), ROWS - 1)][tid];
        if (rb >= 1 && rb < ROWS) t[rb][tid] = t[rb - 1][tid];
    }
    __syncthreads();
}

// vertical column sums of coarse column `col` for the quads of row `row` (lane pairs: two 16-bit lanes per word; the
// largest value, 8 * 255, leaves room for the horizontal pass: 8 * 2040 + 32 < 2^15)
__device__ __forceinline__ void colsum_lanes(const uint2 (*up)[UPS], uint4 (*cs)[UPW], int col, int row)  // col: staged column
{
    const uint2 a0 = up[row][col], a1 = up[row + 1][col], a2 = up[row + 2][col];
    uint4 v;
    v.x = a0.x + a2.x + 6u * a1.x;  // even output row: 1 6 1
    v.y = a1.x + a2.x;              // odd output row: 4 4 (the factor lives in the final shift)
    v.z = a0.y + a2.y + 6u * a1.y;
    v.w = a1.y + a2.y;
    cs[row][col] = v;
}

__device__ __forceinline__ int lane_lo(unsigned v) { return (int)(short)(v & 0xffffu); }
__device__ __forceinline__ int lane_hi(unsigned v) { return (int)v >> 16; }
__device__ __forceinline__ unsigned lanes(int lo, int hi) { return ((unsigned)lo & 0xffffu) | ((unsigned)hi << 16); }
__device__ __forceinline__ int trunc16(float v) { return (int)(short)__float2int_rz(v); }
__device__ __forceinline__ int norm16(int acc, float den, float rr) { return f2s_wrap(fdiv_by((float)(int)(short)acc, den, rr)); }

// n = (short)trunc(a / (wsum + 1e-5)) on two signed 16-bit lanes, for the weight sums that need no division.
// unit (wsum exactly 1, or 0 with a == 0): den = 1 + 84 ulp, the quotient lies strictly between |a| - 1 and |a| and
// truncates to a - sign(a) (proof in sb_collapse_fast.cu; |a| <= 255 here because weights are <= 1).
__device__ __forceinline__ unsigned norm_unit2(unsigned a)
{
    // a - sign(a) = max(a - 1, min(a + 1, 0)): two VIADDMNMX.S16x2
    return __viaddmax_s16x2(a, 0xffffffffu, __viaddmin_s16x2(a, 0x00010001u, 0u));
}
// two (wsum exactly 2): the quotient truncates to (|a| - 1) / 2 rounded toward zero, with the sign of a, i.e.
// floor((a + d) / 2) with d = -1 for a > 0, +2 for a < 0, 0 for a == 0 (|a| <= 510).  The floor of a lane is taken on
// the biased (non-negative) value so that a plain shift + mask serves both lanes.
__device__ __forceinline__ unsigned norm_two2(unsigned a)
{
    const unsigned t = ~a;                                                                 // -a - 1 per lane
    const unsigned d = __viaddmax_s16x2(__viaddmin_s16x2(t, t, 0u), 0x00020002u, 0xffffffffu);  // clamp(-2a, -1, 2) = max(min(2t, 0) + 2, -1)
    const unsigned xb = __vadd2(__vadd2(a, d), 0x04000400u);                                // a + d + 1024 > 0
    return __vadd2((xb >> 1) & 0x7fff7fffu, 0xfe00fe00u);                                   // - 512 per lane
}

template <int LV, bool SLABS>
__global__ void __launch_bounds__(QX *QY, LV == 0 ? 6 : 4) k_collapse_tile(const __grid_constant__ CollapseArgs A)
{
    grid_dependency_sync();
#ifndef SB_EMU
    extern __shared__ __align__(16) unsigned char smem_raw[];
#else
    unsigned char *smem_raw = emu_smem;
#endif
    Smem<LV> &S = *reinterpret_cast<Smem<LV> *>(smem_raw);
    const TileDesc *__restrict__ tile = A.tile;
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * QX + tx;
    const int tile_x = (A.rx0 & ~(TW - 1)) + blockIdx.x * TW, tile_y = A.ry0 + blockIdx.y * TH;  // staged rows start at 16-byte boundaries

    // the collapsed level l+1 around the tile (3 planes x 10 rows x 6 chunks): in flight while the item list is built.
    // Warp ty stages plane-rows 4 ty .. 4 ty + 3, eight lanes per row, six of them with a chunk.
    {
        const int pr = 4 * ty + (tx >> 3), ch = tx & 7;
        if (pr < 3 * UPH && ch < C1S / 8) {
            const int plane = pr >= 2 * UPH ? 2 : (pr >= UPH ? 1 : 0), row = pr - UPH * plane;
            const int xb = 2 * ((tile_x >> 1) - 1 - C1O) + 16 * ch;  // origin 32 k - 8 elements: a 16-byte boundary of an int16 row
            stage_chunk(&S.c1[plane][row][8 * ch], A.up.c + (long long)plane * A.up.plane, 2u * (unsigned)A.up.pitch, (tile_y >> 1) - 1 + row,
                        A.up.h_px, xb, (2 * A.up.w_px + 15) & ~15);
        }
        cp_async_commit();
    }
    // the items whose rect touches this tile, in feed order (warp 0)
    if (ty == 0) {
        int cnt = 0;
        for (int base = 0; base < A.n; base += 32) {
            const int i = base + tx;
            bool c = false;
            if (i < A.n) {
                const int4 r = __ldg(reinterpret_cast<const int4 *>(&tile[i].x0));
                c = tile_x < r.x + r.z && tile_x + TW > r.x && tile_y < r.y + r.w && tile_y + TH > r.y;
            }
            const unsigned m = __ballot_sync(0xffffffffu, c);
            if (c) S.list[cnt + __popc(m & ((1u << tx) - 1u))] = (unsigned short)i;
            cnt += __popc(m);
        }
        if (tx == 0) S.list_n = cnt;
    }
    __syncthreads();
    const int n_cover = S.list_n;

    // all threads: the asynchronous copies of item k's windows into buffer k & 1 (one commit group per item).  Warp ty
    // stages rows 2 ty and 2 ty + 1 of the level-l windows and row ty (warps 0, 1 also rows 8, 9) of the coarse window,
    // lane = chunk: no divisions, one address per thread and window.
    auto stage_item = [&](int k) {
        const int idx = S.list[k];
        const TileDesc &d = tile[idx];
        const ColDesc &cd = A.col[idx];
        if (SLABS && __ldg(&cd.kind) == 1) {  // a slab of partial sums: read directly by the consumers (tile-uniform)
            cp_async_commit();
            return;
        }
        const int4 r = __ldg(reinterpret_cast<const int4 *>(&d.x0));   // x0, y0, w, h
        const int4 o = __ldg(reinterpret_cast<const int4 *>(&d.ox));   // ox, oy, uw, uh
        ItemBuf<LV> &B = S.item[k & 1];
        if constexpr (LV == 0) {
            if (tx < RGS / 4) {
                const int xb = 4 * ((tile_x - r.x) & ~3) + 16 * tx;  // from the 16-byte boundary at or left of the tile
                const int row = tile_y - r.y + 2 * ty;
                const unsigned pb = 4u * (unsigned)cd.rgbm_pitch;
                const int rb = (4 * r.z + 15) & ~15;
                stage_chunk(&B.own[2 * ty][4 * tx], cd.rgbm, pb, row, r.w, xb, rb);
                stage_chunk(&B.own[2 * ty + 1][4 * tx], cd.rgbm, pb, row + 1, r.w, xb, rb);
            }
        } else {
            const int X = tile_x - o.x, row = tile_y - o.y + 2 * ty;  // X even (rect origins below the top level are even)
            {
                const unsigned pb = 8u * (unsigned)cd.pitch;
                const int xb = 8 * X + 16 * tx, rb = (8 * r.z + 15) & ~15;
                stage_chunk(&B.own[2 * ty][2 * tx], cd.q, pb, row, r.w, xb, rb);
                stage_chunk(&B.own[2 * ty + 1][2 * tx], cd.q, pb, row + 1, r.w, xb, rb);
            }
            if (tx < RGS / 4) {
                const unsigned pb = 4u * (unsigned)cd.pitch;
                const int xb = 4 * (X & ~3) + 16 * tx, rb = (4 * r.z + 15) & ~15;
                stage_chunk(&B.w[2 * ty][4 * tx], cd.w, pb, row, r.w, xb, rb);
                stage_chunk(&B.w[2 * ty + 1][4 * tx], cd.w, pb, row + 1, r.w, xb, rb);
            }
        }
        if (tx < UPS / 2) {
            const int bx = (((tile_x - o.x) >> 1) - 1) & ~1, by = ((tile_y - o.y) >> 1) - 1;  // the even column at or left of the origin
            const unsigned pb = 8u * (unsigned)cd.upitch;
            const int xb = 8 * bx + 16 * tx, rb = (8 * o.z + 15) & ~15;
            stage_chunk(&B.up[ty][2 * tx], cd.uq, pb, by + ty, o.w, xb, rb);
            if (ty < UPH - QY) stage_chunk(&B.up[QY + ty][2 * tx], cd.uq, pb, by + QY + ty, o.w, xb, rb);
        }
        cp_async_commit();
    };
    if (n_cover > 0) stage_item(0);

    // accumulators of the quad (index dy * 2 + dx): red | blue << 16 as two wrap-around lanes, green, weight sum
    unsigned acc_rb[4] = {0u, 0u, 0u, 0u};
    int acc_g[4] = {0, 0, 0, 0};
    float wsum[4] = {0.f, 0.f, 0.f, 0.f};

    for (int k = 0; k < n_cover; ++k) {
        // item k+1 goes into the other buffer, whose last reader passed the second barrier of iteration k-1
        if (k + 1 < n_cover) {
            stage_item(k + 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();  // item k's windows (and C_{l+1}'s) are complete for every thread
        ItemBuf<LV> &B = S.item[k & 1];
        const TileDesc &d = tile[S.list[k]];
        if (SLABS) {
            const ColDesc &cd = A.col[S.list[k]];
            if (__ldg(&cd.kind) == 1) {
                // partial sums of another rank over (part of) this tile: int16 wrap-around adds, the float weight sum in
                // item order (= rank order); rect origins and sizes are even: a quad is in or out as a whole
                const int4 r = __ldg(reinterpret_cast<const int4 *>(&cd.ox));  // ox, oy, w_l, h_l
                const int X = tile_x + 2 * tx - r.x, Y = tile_y + 2 * ty - r.y;
                if ((unsigned)X < (unsigned)r.z && (unsigned)Y < (unsigned)r.w) {
                    const int pitch = __ldg(&cd.pitch), plane = __ldg(&cd.plane);
                    const int16_t *g = cd.g;
                    const float *w = cd.w;
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int o = (Y + (q >> 1)) * pitch + X + (q & 1);
                        acc_rb[q] = __vadd2(acc_rb[q], lanes(g[o], g[2 * plane + o]));
                        acc_g[q] += g[plane + o];
                        wsum[q] = fadd(wsum[q], w[o]);
                    }
                }
                continue;  // (tile-uniform: no thread waits at the second barrier of this iteration)
            }
        }
        const int4 o = __ldg(reinterpret_cast<const int4 *>(&d.ox));  // ox, oy, uw, uh
        const int bx = ((tile_x - o.x) >> 1) - 1, by = ((tile_y - o.y) >> 1) - 1;
        const int su = bx & 1;  // logical column c of the coarse window = staged column c + su
        if (bx < 0 || by < 0 || bx + UPW > o.z || by + UPH > o.w)
            fix_borders<uint2, UPH, UPW, UPS>(reinterpret_cast<uint2(*)[UPS]>(&B.up[0][su]), bx, by, o.z, o.w, tid);
        uint4(*cs)[UPW] = S.cs[k & 1];
        {
            const uint2(*ups)[UPS] = reinterpret_cast<const uint2(*)[UPS]>(&B.up[0][su]);
            colsum_lanes(ups, cs, tx, ty);
            if (tid < 2 * QY) colsum_lanes(ups, cs, QX + (tid & 1), tid >> 1);  // the two columns right of the last quad
        }

        // the quad's own pixels: g_rb = r | b << 16, g_g = green, wt = weight
        unsigned g_rb[4], g_g[4];
        float wt[4];
        bool nothing, unit;
        if constexpr (LV == 0) {
            const int sx = ((tile_x - __ldg(&d.x0)) & 3) + 2 * tx;  // the staged window starts at a multiple of 4 pixels
            const unsigned p[4] = {B.own[2 * ty][sx], B.own[2 * ty][sx + 1], B.own[2 * ty + 1][sx], B.own[2 * ty + 1][sx + 1]};
            nothing = ((p[0] | p[1] | p[2] | p[3]) >> 24) == 0u;           // all four weights are exactly 0
            unit = ((p[0] & p[1] & p[2] & p[3]) >> 24) == 255u;             // all four weights are exactly 1
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                g_rb[q] = p[q] & 0x00ff00ffu;
                g_g[q] = (p[q] >> 8) & 255u;
                wt[q] = unit ? 1.f : fmul((float)(p[q] >> 24), SB_INV255);  // 255 * fl(1/255) == 1 exactly
            }
        } else {
            const int sw = ((tile_x - o.x) & 3) + 2 * tx;  // the staged weight window starts at a multiple of 4 columns
            const float2 w0 = *reinterpret_cast<const float2 *>(&B.w[2 * ty][sw]);
            const float2 w1 = *reinterpret_cast<const float2 *>(&B.w[2 * ty + 1][sw]);
            const uint4 a = *reinterpret_cast<const uint4 *>(&B.own[2 * ty][2 * tx]);
            const uint4 b = *reinterpret_cast<const uint4 *>(&B.own[2 * ty + 1][2 * tx]);
            wt[0] = w0.x; wt[1] = w0.y; wt[2] = w1.x; wt[3] = w1.y;
            g_rb[0] = a.x; g_g[0] = a.y; g_rb[1] = a.z; g_g[1] = a.w;
            g_rb[2] = b.x; g_g[2] = b.y; g_rb[3] = b.z; g_g[3] = b.w;
            nothing = wt[0] == 0.f && wt[1] == 0.f && wt[2] == 0.f && wt[3] == 0.f;
            unit = wt[0] == 1.f && wt[1] == 1.f && wt[2] == 1.f && wt[3] == 1.f;
        }
        __syncthreads();        // the column sums of this image are complete
        if (nothing) continue;  // (short)trunc(L * 0) == 0 and wsum + 0 == wsum: contributes exactly nothing

        // pyrUp of the image's level l+1 at the four pixels: horizontal pass over the three column sums
        const uint4 c0 = cs[ty][tx], c1 = cs[ty][tx + 1], c2 = cs[ty][tx + 2];
        const unsigned M = 0x00ff00ffu;
        unsigned u_rb[4], u_g[4];
        u_rb[0] = ((c0.x + c2.x + 6u * c1.x + 0x00200020u) >> 6) & M;
        u_rb[1] = ((c1.x + c2.x + 0x00080008u) >> 4) & M;
        u_rb[2] = ((c0.y + c2.y + 6u * c1.y + 0x00080008u) >> 4) & M;
        u_rb[3] = ((c1.y + c2.y + 0x00020002u) >> 2) & M;
        u_g[0] = (c0.z + c2.z + 6u * c1.z + 32u) >> 6;
        u_g[1] = (c1.z + c2.z + 8u) >> 4;
        u_g[2] = (c0.w + c2.w + 6u * c1.w + 8u) >> 4;
        u_g[3] = (c1.w + c2.w + 2u) >> 2;
        if (unit) {  // (short)trunc(L * 1.0f) == L
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                acc_rb[q] = __vadd2(acc_rb[q], __vsub2(g_rb[q], u_rb[q]));
                acc_g[q] += (int)g_g[q] - (int)u_g[q];
                wsum[q] = fadd(wsum[q], 1.f);
            }
        } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const unsigned lap_rb = __vsub2(g_rb[q], u_rb[q]);
                const int lap_g = (int)g_g[q] - (int)u_g[q];
                const int tr = trunc16(fmul((float)lane_lo(lap_rb), wt[q]));
                const int tb = trunc16(fmul((float)lane_hi(lap_rb), wt[q]));
                acc_rb[q] = __vadd2(acc_rb[q], lanes(tr, tb));
                acc_g[q] += trunc16(fmul((float)lap_g, wt[q]));
                wsum[q] = fadd(wsum[q], wt[q]);
            }
        }
    }

    // ---- pyrUp of the collapsed level l+1 ---------------------------------------------------------------------------
    if (n_cover == 0) {
        cp_async_wait<0>();
        __syncthreads();
    }
    {
        const int bx = (tile_x >> 1) - 1, by = (tile_y >> 1) - 1;
        if (bx < 0 || by < 0 || bx + UPW > A.up.w_px || by + UPH > A.up.h_px) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
                fix_borders<int16_t, UPH, UPW, C1S>(reinterpret_cast<int16_t(*)[C1S]>(&S.c1[c][0][C1O]), bx, by, A.up.w_px, A.up.h_px, tid);
        }
    }
    __syncthreads();  // nobody reads the images' column sums any more: the buffers now take those of C_{l+1}
    int4(*csa)[UPW] = reinterpret_cast<int4(*)[UPW]>(S.cs[0]);   // e_r, e_g, e_b, o_r
    int2(*csb)[UPW] = reinterpret_cast<int2(*)[UPW]>(S.cs[1]);   // o_g, o_b
    auto colsum_c = [&](int col, int row) {
        int e[3], od[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int a0 = S.c1[c][row][col + C1O], a1 = S.c1[c][row + 1][col + C1O], a2 = S.c1[c][row + 2][col + C1O];
            e[c] = a0 + a2 + 6 * a1;
            od[c] = a1 + a2;
        }
        csa[row][col] = make_int4(e[0], e[1], e[2], od[0]);
        csb[row][col] = make_int2(od[1], od[2]);
    };
    colsum_c(tx, ty);
    if (tid < 2 * QY) colsum_c(QX + (tid & 1), tid >> 1);
    __syncthreads();
    int u[3][4];  // [channel][pixel of the quad]
    {
        const int4 a0 = csa[ty][tx], a1 = csa[ty][tx + 1], a2 = csa[ty][tx + 2];
        const int2 b0 = csb[ty][tx], b1 = csb[ty][tx + 1], b2 = csb[ty][tx + 2];
        const int e0[3] = {a0.x, a0.y, a0.z}, e1[3] = {a1.x, a1.y, a1.z}, e2[3] = {a2.x, a2.y, a2.z};
        const int o0[3] = {a0.w, b0.x, b0.y}, o1[3] = {a1.w, b1.x, b1.y}, o2[3] = {a2.w, b2.x, b2.y};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            u[c][0] = (e0[c] + e2[c] + 6 * e1[c] + 32) >> 6;
            u[c][1] = (e1[c] + e2[c] + 8) >> 4;
            u[c][2] = (o0[c] + o2[c] + 6 * o1[c] + 8) >> 4;
            u[c][3] = (o1[c] + o2[c] + 2) >> 2;
        }
    }

    const int x = tile_x + 2 * tx, y = tile_y + 2 * ty;  // top-left pixel of the quad
    if (x < A.rx0 || x >= A.rx0 + A.rw || y >= A.ry0 + A.rh) return;  // (after the last barrier)

    // ---- blend step on lanes: words [row][0] = pixel 0 (r | b << 16), [row][1] = pixel 1, [row][2] = green of both ------
    unsigned N[2][3];
    const bool unit = (wsum[0] == 1.f || wsum[0] == 0.f) && (wsum[1] == 1.f || wsum[1] == 0.f) && (wsum[2] == 1.f || wsum[2] == 0.f) &&
                      (wsum[3] == 1.f || wsum[3] == 0.f);
    const bool two = wsum[0] == 2.f && wsum[1] == 2.f && wsum[2] == 2.f && wsum[3] == 2.f;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
        N[dy][0] = acc_rb[2 * dy];
        N[dy][1] = acc_rb[2 * dy + 1];
        N[dy][2] = __byte_perm((unsigned)acc_g[2 * dy], (unsigned)acc_g[2 * dy + 1], 0x5410);
    }
    if (unit) {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int j = 0; j < 3; ++j) N[dy][j] = norm_unit2(N[dy][j]);
    } else if (two) {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int j = 0; j < 3; ++j) N[dy][j] = norm_two2(N[dy][j]);
    } else {  // fractional weight sums: one refined reciprocal per pixel, an exact quotient per channel (sb_device.cuh)
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
            int n[2][3];
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const float den = fadd(wsum[2 * dy + dx], SB_WEIGHT_EPS);
                const float rr = rcp_refined(den);
                n[dx][0] = norm16(lane_lo(N[dy][dx]), den, rr);
                n[dx][1] = norm16(dx ? lane_hi(N[dy][2]) : lane_lo(N[dy][2]), den, rr);
                n[dx][2] = norm16(lane_hi(N[dy][dx]), den, rr);
            }
            N[dy][0] = lanes(n[0][0], n[0][2]);
            N[dy][1] = lanes(n[1][0], n[1][2]);
            N[dy][2] = lanes(n[0][1], n[1][1]);
        }
    }
    // collapse add: |pyrUp| <= 256 (nb - l) and |n| <= 255 for byte-fed images, far inside int16: the lane-wise
    // wrap-around add equals the reference's saturating add
    unsigned V[2][3];
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
        V[dy][0] = __vadd2(N[dy][0], lanes(u[0][2 * dy], u[2][2 * dy]));
        V[dy][1] = __vadd2(N[dy][1], lanes(u[0][2 * dy + 1], u[2][2 * dy + 1]));
        V[dy][2] = __vadd2(N[dy][2], lanes(u[1][2 * dy], u[1][2 * dy + 1]));
    }
    if (LV == 1) {  // C_l: three int16 planes, two pixels per 4-byte store
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
            const int o = (y + dy) * A.cur.pitch + x;
            *reinterpret_cast<unsigned *>(A.cur.c + o) = __byte_perm(V[dy][0], V[dy][1], 0x5410);
            *reinterpret_cast<unsigned *>(A.cur.c + A.cur.plane + o) = V[dy][2];
            *reinterpret_cast<unsigned *>(A.cur.c + 2 * A.cur.plane + o) = __byte_perm(V[dy][0], V[dy][1], 0x7632);
        }
        return;
    }
    // level 0: mask, zero outside it, |v| saturated to uint8 (convertScaleAbs), crop to the roi
    const PanoOut &out = A.out;
    const unsigned xo = (unsigned)(x - A.out_x0);
    unsigned o_rgb = (unsigned)y * (unsigned)out.rgb_pitch + 3u * xo, o_m = (unsigned)y * (unsigned)out.mask_pitch + xo;
    const bool both = x >= A.out_lo && x + 1 < A.out_hi;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
        if (y + dy < out.h) {
            const unsigned m0 = wsum[2 * dy] > SB_WEIGHT_EPS ? 0xffffffffu : 0u, m1 = wsum[2 * dy + 1] > SB_WEIGHT_EPS ? 0xffffffffu : 0u;
            unsigned Bq[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) Bq[j] = __vmins2(__viaddmax_s16x2(~V[dy][j], 0x00010001u, V[dy][j]), 0x00ff00ffu);  // min(max(-v, v), 255)
            Bq[0] &= m0;
            Bq[1] &= m1;
            Bq[2] &= __byte_perm(m0, m1, 0x5410);
            // bytes r0 g0 | b0 r1 | g1 b1
            const unsigned h0 = __byte_perm(Bq[0], Bq[2], 0x0040), h1 = __byte_perm(Bq[0], Bq[1], 0x0042), h2 = __byte_perm(Bq[2], Bq[1], 0x0062);
            const unsigned hm = __byte_perm(m0, m1, 0x0040);
            if (both) {
                unsigned short *p2 = reinterpret_cast<unsigned short *>(out.rgb + o_rgb);
                p2[0] = (unsigned short)h0;
                p2[1] = (unsigned short)h1;
                p2[2] = (unsigned short)h2;
                *reinterpret_cast<unsigned short *>(out.mask + o_m) = (unsigned short)hm;
            } else {  // the roi's last (odd) column, or a column outside [out_lo, out_hi)
                if (x >= A.out_lo && x < A.out_hi) {
                    out.rgb[o_rgb] = (uint8_t)h0;
                    out.rgb[o_rgb + 1] = (uint8_t)(h0 >> 8);
                    out.rgb[o_rgb + 2] = (uint8_t)h1;
                    out.mask[o_m] = (uint8_t)hm;
                }
                if (x + 1 >= A.out_lo && x + 1 < A.out_hi) {
                    out.rgb[o_rgb + 3] = (uint8_t)(h1 >> 8);
                    out.rgb[o_rgb + 4] = (uint8_t)h2;
                    out.rgb[o_rgb + 5] = (uint8_t)(h2 >> 8);
                    out.mask[o_m + 1] = (uint8_t)(hm >> 8);
                }
            }
        }
        o_rgb += (unsigned)out.rgb_pitch;
        o_m += (unsigned)out.mask_pitch;
    }
}

}  // namespace

bool collapse_tile_enabled()
{
#ifdef SB_EMU
    return getenv("SB_EMU_BLOCKS") != nullptr;  // one host thread per thread of a CTA: correct but slow, on request only
#else
    static const bool on = [] {
        const char *e = getenv("SB_TILE");
        return !(e && e[0] == '0');
    }();
    return on;
#endif
}

int launch_collapse_tile(const CollapseArgs &A, int l, int nb, cudaStream_t s)
{
    // levels 0 and 1 only: from level 2 on the levels are small and the per-tile staging overhead outweighs what it
    // saves (SB_TILE_MAXL overrides)
    static const int max_level = [] {
        const char *e = getenv("SB_TILE_MAXL");
        return e ? atoi(e) : 1;
    }();
    if (!A.tile || l >= nb || l > max_level || A.partial || A.n > SB_MAX_ITEMS || !collapse_tile_enabled()) return SB_ERR_STATE;
    if ((A.rx0 | A.ry0 | A.rw | A.rh) & 1) return SB_ERR_STATE;
    if (l == 0) {
        const PanoOut &out = A.out;
        const bool plain = out.rgb && out.mask && !out.s16 && ((out.rgb_pitch | out.mask_pitch | A.out_x0) & 1) == 0 &&
                           out.rgb_pitch * out.h < (1ll << 32);
        if (!plain) return SB_ERR_STATE;
    } else if ((long long)A.cur.plane * 3 >= (1ll << 31)) {
        return SB_ERR_STATE;
    }
    if (A.rw <= 0 || A.rh <= 0) return SB_OK;
#ifndef SB_EMU
    static bool attr_set = false;
    if (!attr_set) {
        SB_CUDA(cudaFuncSetAttribute(k_collapse_tile<0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem<0>)));
        SB_CUDA(cudaFuncSetAttribute(k_collapse_tile<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem<1>)));
        SB_CUDA(cudaFuncSetAttribute(k_collapse_tile<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem<0>)));
        SB_CUDA(cudaFuncSetAttribute(k_collapse_tile<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem<1>)));
        attr_set = true;
    }
#endif
    dim3 block(QX, QY), grid(div_up(A.rx0 + A.rw - (A.rx0 & ~(TW - 1)), TW), div_up(A.rh, TH));
#ifdef SB_EMU
    if (getenv("SB_EMU_TRACE")) fprintf(stderr, "k_collapse_tile<%d, %d> %ux%u tiles, %d items\n", l, A.has_slabs, grid.x, grid.y, A.n);
#endif
    if (l == 0 && A.has_slabs)
        launch_block(k_collapse_tile<0, true>, grid, block, sizeof(Smem<0>), s, A);
    else if (l == 0)
        launch_block(k_collapse_tile<0, false>, grid, block, sizeof(Smem<0>), s, A);
    else if (A.has_slabs)
        launch_block(k_collapse_tile<1, true>, grid, block, sizeof(Smem<1>), s, A);
    else
        launch_block(k_collapse_tile<1, false>, grid, block, sizeof(Smem<1>), s, A);
    return launch_check("k_collapse_tile");
}


}  // namespace sb
