// Shared machinery of the forward and backward composite kernels (persistent, warp-specialised).
//
// The reference renders one 16x16 tile per 256-thread block, every thread doing everything
// (forward.cu:261-396).  Here a persistent CTA pulls tiles from an atomic counter and splits the
// work over warp roles that talk only through shared-memory rings + mbarriers:
//
//   producer group (4)    warp 0 walks the tile's slice of the depth-sorted instance list, drops the
//                         instances whose alpha >= 1/255 footprint cannot reach the tile, and fills
//                         a ring of stages with 48-byte splat records.  The records reach it through a
//                         small shared-memory queue (RecQueue) that cp.async fills kPrefetch chunks of 32
//                         ahead of the cull, across the boundary to the next tile.  When there
//                         are features, warp 1 (the copy warp) fetches the stage's C-wide feature
//                         rows (float32 or float16: the ring's element type TF) with 1-D TMA bulk
//                         copies (cp.async.bulk -> UBLKCP) that complete on the stage's `full` mbarrier.  The producer runs ahead across tile
//                         boundaries, so the next tile's first stage is already resident when the
//                         consumers get there (no per-tile start-up bubble).  Warps 2 and 3 retire.
//   alpha warps (8)       warp a owns the 8x4 pixel block a of the tile, one pixel per lane: alpha,
//                         the T recurrence, RGB/depth (and in the backward every geometric gradient
//                         term).  In the forward they publish the blend weights w = alpha*T as a
//                         [instance][pixel] tile plus a per-instance pixel mask in a small per-block
//                         ring (`wfull`/`wempty`), and per 8x2 half of the block a mask of the
//                         instances that blended a pixel there.
//   feature warps (16)    forward only: a pair per block.  Warp h of block b's pair owns rows 2h and
//                         2h+1 of the block (quads 4h..4h+3, pixel-mask bits 16h..16h+15) and consumes
//                         the entries of block b's weight tiles that blended a pixel of that half, with
//                         one float4 of channels per lane; the half's 16 pixels x 4 channels stay in
//                         registers, and the weights arrive as broadcast LDS.128 per 2x2 pixel quad.
//
// The forward with features launches all 28 warps (composite_fwd.cu; without features, 20 warps with no feature warp
// doing any work); the backward geometry kernel launches the producer group and the alpha warps only (composite_bwd.cu).
#pragma once
#include <initializer_list>

#include "kernels.h"

namespace f3dgs {

constexpr int kBlocksPerTile = 8;   // 8x4-pixel blocks in a 16x16 tile
constexpr int kProducerWarp = 0;    // warps 0..3: producer warpgroup
constexpr int kAlphaWarp0 = 4;      // then one alpha warp per pixel block
constexpr int kAlphaWarps = kBlocksPerTile;
constexpr int kFeatWarp0 = kAlphaWarp0 + kAlphaWarps;  // then two feature warps per pixel block (forward)
constexpr int kRegsProducer = 40;   // setmaxnreg of the producer group
constexpr int kStageEntries = 32;
constexpr int kStages = 6;
constexpr int kWSlots = 2;
constexpr int kDoneSlots = 8;       // > kStages: the producer is never further ahead than that.  Slots are indexed by the
                                    // CTA's own work sequence number, NOT by the work id: ids come from a global
                                    // atomic counter, so two items in flight in one CTA can be congruent mod 8.

// TF: element type of the staged feature rows, float or __half (a float16 row is half the bytes)
template <int CH, typename TF = float>
struct alignas(128) Stage {
    TF feat[CH > 0 ? kStageEntries : 1][CH > 0 ? CH : 4];  // CH == 0: dummy, never touched
    float4 rec0[kStageEntries];                   // x, y, ex, ey
    float4 rec1[kStageEntries];                   // conic a, b, c, opacity
    float4 rec2[kStageEntries];                   // r, g, b, depth
    uint32_t listpos[kStageEntries];              // 1-based position in the tile's list (reference `contributor`)
    uint32_t gid[kStageEntries];                  // Gaussian index
    uint32_t n;                                   // valid entries
    uint32_t last;                                // 1 = last stage of this work item
    uint32_t first;                               // 1 = first stage of this work item
    int32_t work;                                 // work item (tile * chunks + chunk); < 0: no more work
    uint32_t done_slot;                           // index into RingV2::done_mask for this work item
};

struct alignas(128) WSlot {
    float w[kStageEntries][32];    // blend weights [instance][pixel of the block]
    uint32_t pm[kStageEntries];    // per instance: which pixels blended
    uint32_t km[2];                // km[h]: which instances blended a pixel of rows 2h, 2h+1 (pm bits 16h..16h+15)
    uint32_t last;
    uint32_t first;
    int32_t work;
};
static_assert(sizeof(WSlot) == 4352, "weight slot layout changed");  // 4244 bytes of fields, padded to 128

// The producer's record queue: splat records on their way from global memory to the producer warp, kPrefetch chunks of
// 32 records, filled by cp.async (in-flight copies hold no registers) and read back by the lane that issued the copy.
constexpr int kPrefetch = 4;
struct alignas(16) RecQueue {
    float4 q[kPrefetch][3][32];  // [slot][16-byte third of the 48-byte record][lane]
    uint32_t id[kPrefetch][32];  // Gaussian index
};

// WB x WJ: dimensions of the weight-slot ring (pixel blocks x slots per block)
template <int CH, typename TF = float, int WB = kBlocksPerTile, int WJ = kWSlots>
struct alignas(128) RingV2 {
    using Feat = TF;
    static constexpr int kWB = WB, kWJ = WJ;
    Stage<CH, TF> stage[kStages];
    WSlot ws[WB][WJ];
    uint64_t full[kStages];
    uint64_t empty[kStages];
    uint64_t listed[kStages];  // records + ids of the stage are written: the copy warp may fetch its feature rows
    uint64_t wfull[WB][WJ];
    uint64_t wempty[WB][WJ];
    uint32_t done_mask[kDoneSlots];  // bit b set: pixel block b of that work item needs no more instances
    RecQueue rq;                     // private to the producer warp: no barrier guards it
};

// The ring without feature rows and with a single weight slot, for the backward geometry kernel, which has no feature
// warps: 22 KB instead of 86 KB of shared memory, so that two CTAs fit on an SM.  The one-element `ws` / `wfull` /
// `wempty` are not used; ring_init<> initialises the two barriers.
using RingSlim = RingV2<0, float, 1, 1>;

static_assert(sizeof(RecQueue) == 6656, "record queue layout changed");
static_assert(sizeof(RingV2<0>) == 88320 && sizeof(RingSlim) == 22784, "ring layout changed");
static_assert(sizeof(RingV2<32>) == 112896 && sizeof(RingV2<64>) == 137472 && sizeof(RingV2<128>) == 186624,
              "ring layout changed");
static_assert(sizeof(RingV2<32, __half>) == 100608 && sizeof(RingV2<64, __half>) == 112896 &&
                  sizeof(RingV2<128, __half>) == 137472,
              "ring layout changed");

// ---------------------------------------------------------------- pixel-block layout
// A 16x16 tile is 8 blocks of 8x4 pixels, 2 across and 4 down.  Slot p of a block (an alpha warp's lane, a column of
// the weight tiles and of the emitted list_w rows) is pixel i = p & 3 of the 2x2 quad q = p >> 2; the quads lie 4
// across, so bits 4q..4q+3 of a pixel mask are quad q.
// Origin (bx0, by0) of block b of the tile at (tile_x, tile_y); tile = tile_y * tiles_x + tile_x.
__device__ __forceinline__ int block_x0(int tile_x, int b) { return tile_x * 16 + (b & 1) * 8; }
__device__ __forceinline__ int block_y0(int tile_y, int b) { return tile_y * 16 + (b >> 1) * 4; }
// offset of slot p from the block origin
__device__ __forceinline__ int slot_px(int p) { return ((p >> 2) & 3) * 2 + (p & 1); }
__device__ __forceinline__ int slot_py(int p) { return (p >> 4) * 2 + ((p >> 1) & 1); }

// Register tile of a feature lane: float2 t[NQ][2][4] = [quad][quad row][channel], the two pixels of a quad row in .x
// and .y (one paired FMA covers both).  With CH / 4 lanes per feature row, G = 32 / (CH / 4) lane groups share the
// tile's quads (8 for a whole block, 4 for an 8x2 half): group grp holds quads qi * G + grp, qi < NQ = 8 / G (or 4 / G).
template <int NQ>
__device__ __forceinline__ float& tile_px(float2 (&t)[NQ][2][4], int qi, int i, int c) {
    return (i & 1) ? t[qi][i >> 1][c].y : t[qi][i >> 1][c].x;
}
// Pixel k of the run of pixels 4 * half .. 4 * half + 3 in row y of the register tile, for a lane that holds all its quads
// (G == 1).  (% NQ only keeps the indices in range in the instantiations with G > 1, which never get here.)
template <int NQ>
__device__ __forceinline__ float& tile_run_px(float2 (&t)[NQ][2][4], int y, int half, int k, int c) {
    return tile_px(t, ((y >> 1) * 4 + half * 2 + (k >> 1)) % NQ, (y & 1) * 2 + (k & 1), c);
}
template <int NQ>
__device__ __forceinline__ float4 tile_run(float2 (&t)[NQ][2][4], int y, int half, int c) {
    return make_float4(tile_run_px(t, y, half, 0, c), tile_run_px(t, y, half, 1, c), tile_run_px(t, y, half, 2, c),
                       tile_run_px(t, y, half, 3, c));
}
template <int NQ>
__device__ __forceinline__ void set_tile_run(float2 (&t)[NQ][2][4], int y, int half, int c, float4 v) {
    tile_run_px(t, y, half, 0, c) = v.x;
    tile_run_px(t, y, half, 1, c) = v.y;
    tile_run_px(t, y, half, 2, c) = v.z;
    tile_run_px(t, y, half, 3, c) = v.w;
}

// Visits one channel plane of a register tile over the block's pixels inside the W x H image, in the widest access the
// plane allows, and hands each access its address in `plane`:
//   row(p, y)           8-pixel row y: G == 1, `rows` (8-pixel alignment of the plane) and the row inside the image
//   run(p, y, half)     4-pixel run: G == 1 and `runs` (4-pixel alignment)
//   px(p, qi, i)        otherwise pixel i of the lane's quad qi, one at a time
// NY: rows of the register tile, image rows by0 .. by0 + NY - 1.  NY = 2 is one 8x2 half of a block (quads 0..3 of the
// register tile, NQ * G = 4), with by0 the half's first row.
template <int G, int NQ, int NY = 4, typename T, class Row, class Run, class Px>
__device__ __forceinline__ void for_tile_pixels(T* plane, int bx0, int by0, int W, int H, int grp, bool rows, bool runs,
                                                Row row, Run run, Px px) {
    static_assert(NQ * G * 2 == NY * 4, "a register tile of NQ quads per lane group covers NY rows of 8 pixels");
    if (G == 1 && rows && bx0 + 8 <= W) {
#pragma unroll
        for (int y = 0; y < NY; y++) {
            const int yy = by0 + y;
            if (yy >= H) continue;
            row(plane + (size_t)yy * W + bx0, y);
        }
    } else if (G == 1 && runs) {
#pragma unroll
        for (int y = 0; y < NY; y++) {
            const int yy = by0 + y;
            if (yy >= H) continue;
#pragma unroll
            for (int half = 0; half < 2; half++) {
                const int xx = bx0 + half * 4;
                if (xx >= W) continue;
                run(plane + (size_t)yy * W + xx, y, half);
            }
        }
    } else {
#pragma unroll
        for (int qi = 0; qi < NQ; qi++) {
            const int q = qi * G + grp;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                // slot_px / slot_py of slot 4 * q + i, spelled per quad: q is a runtime value when G > 1, and the compiler
                // does not fold slot_px(4 * q + i) back to this form (280-460 more SASS instructions in each CH = 32 / 64
                // forward kernel)
                const int xx = bx0 + (q & 3) * 2 + (i & 1), yy = by0 + (q >> 2) * 2 + (i >> 1);
                if (xx < W && yy < H) px(plane + (size_t)yy * W + xx, qi, i);
            }
        }
    }
}

// Four float16 values (8 bytes, low half first) as float32, exactly
__device__ __forceinline__ float4 to_float4(float4 v) { return v; }
__device__ __forceinline__ float4 to_float4(uint2 v) {
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
    return make_float4(a.x, a.y, b.x, b.y);
}

// ---------------------------------------------------------------- the backward's per-(tile, block) instance lists
// The geometry kernel (composite_bwd.cu, EMIT and LIFT) writes one entry per instance that blended in an 8x4 block, back
// to front; feature_bwd.cu reads them.  An entry is the 32 blend weights w = alpha * T of the block's pixel slots plus
// {Gaussian id, pixel mask}: 136 bytes.
struct InstanceLists {
    float* w;       // [8R][32] blend weights, entry e at w[e * 32 + slot]
    uint2* meta;    // [8R]     {Gaussian id, pixel mask}
    uint32_t* cnt;  // [8 tiles] entries written per (tile, block)
};

// The lists need no counting pass: block b of a tile owns entries [list_begin(range.x, range.y, b), ... + len),
// len = range.y - range.x, because an instance of the tile's list appears at most once per block.  The tiles' ranges
// partition [0, R), so block b's entries end at 8 range.x + (b + 1) len <= 8 range.y <= 8R: a capacity of 8R entries
// (ListLayout) holds every block of every tile.
__device__ __forceinline__ size_t list_begin(uint32_t begin, uint32_t end, int b) {
    return kBlocksPerTile * (size_t)begin + (size_t)b * (end - begin);
}

// Byte offsets of the three lists in one allocation of `bytes`, for R instances over `tiles` tiles
struct ListLayout {
    size_t w, meta, cnt, bytes;
    ListLayout(size_t R, size_t tiles) {
        size_t o = 0;
        w = o;     o = align_up(o + kBlocksPerTile * R * 32 * sizeof(float));
        meta = o;  o = align_up(o + kBlocksPerTile * R * sizeof(uint2));
        cnt = o;   o = align_up(o + kBlocksPerTile * tiles * sizeof(uint32_t));
        bytes = o;
    }
};

// Work counters of the persistent composite kernels: int slots of the 256-byte counter region of the image buffer, for
// composite_fwd.cu, composite_bwd.cu and feature_bwd.cu.  Each launcher takes the region's base and zeroes its own slot.
constexpr int kCounterFwd = 0, kCounterBwdGeom = 16, kCounterFeatureBwd = 48;

// ---- feature_bwd.cu: dL/dfeature[g] += sum over the pixels of each list entry of w * dL/dfeature_map, over the lists of
// the view.  TG (float or __half) is the element type of the map; a __half map stands for dL/dO = scale * float(h) (the
// scale is not read for a float map).  Feature lifting passes the teacher map at scale 1.
template <typename TG>
cudaError_t launch_feature_bwd(const ViewParams& vp, const uint2* ranges, const InstanceLists& lists,
                               const TG* dL_dfeat_pix, float dL_dfeat_pix_scale, float* dL_dfeature, int* counters,
                               cudaStream_t s);
// ---- feature_bwd.cu: overwrites each list entry's weight row with the pair dot products d_ip = f_i . dL/dfeature_map[:, p]
// over the C channels (TG and scale as above), for the FEAT walk of composite_bwd.cu
template <typename TG>
cudaError_t launch_feature_dot(const ViewParams& vp, const uint2* ranges, const InstanceLists& lists,
                               const FeatureRows& feat, const TG* dL_dfeat_pix, float dL_dfeat_pix_scale, int* counters,
                               cudaStream_t s);

// Splat alpha at pixel (pxf, pyf), with the reference's expression trees (forward.cu:340-351, backward.cu:525-535): plain
// fp32, no _rn intrinsics (see common.cuh).  alpha is 0 where the reference skips the pair (power > 0 or alpha < 1/255)
// and where !valid.
struct SplatAlpha {
    float dx, dy, G, alpha;
};
__device__ __forceinline__ SplatAlpha splat_alpha(const float4 r0, const float4 r1, float pxf, float pyf, bool valid) {
    SplatAlpha s;
    s.dx = r0.x - pxf;
    s.dy = r0.y - pyf;
    const float power = -0.5f * (r1.x * s.dx * s.dx + r1.z * s.dy * s.dy) - r1.y * s.dx * s.dy;
    s.G = expf(power);
    const float av = fminf(0.99f, r1.w * s.G);
    s.alpha = (valid && !(power > 0.0f) && !(av < 1.0f / 255.0f)) ? av : 0.f;
    return s;
}

// Can the region where alpha >= 1/255 reach the pixel rectangle [x0,x1] x [y0,y1] (pixel-centre coordinates)?
// r0 = {x, y, ex, ey}, r1 = {conic a, b, c, opacity} of the splat record.  Conservative in both steps: a pair this returns
// false for fails the reference's blend conditions (forward.cu:344-352: power <= 0 and alpha >= 1/255) at every pixel of the
// rectangle, so skipping it cannot change a result.
//   bounding box   the half extents ex, ey stored by the forward preprocess (preprocess.cu: alpha_extent)
//   exact          the minimum over the rectangle of q(d) = a dx^2 + 2 b dx dy + c dy^2 (= -2 power) against
//                  tau = 2.02 ln(255 op) + 0.02 >= 2 ln(255 op).  q is convex (alpha_extent marks indefinite or
//                  ill-conditioned conics "never cull", ex = 3e38), so the minimum is 0 if the centre lies inside and
//                  otherwise sits on one of the four edges, where it is a clamped 1-D parabola.  Removes ~13% of the
//                  (8x4 block, instance) pairs and ~5% of the (tile, instance) pairs the box lets through at configs
//                  2 and 3; tools/check_exact_cull.py restates it in float32 numpy and checks it never drops a needed pair.
__device__ __forceinline__ bool footprint_hits_rect(const float4 r0, const float4 r1, float x0, float x1, float y0,
                                                    float y1) {
    const bool box = (r0.x + r0.z >= x0) && (r0.x - r0.z <= x1) && (r0.y + r0.w >= y0) && (r0.y - r0.w <= y1);
    if (!box) return false;
    const float dxl = r0.x - x1, dxh = r0.x - x0, dyl = r0.y - y1, dyh = r0.y - y0;  // ranges of d over the rectangle
    if (r0.z > 1.0e30f || (dxl <= 0.f && dxh >= 0.f && dyl <= 0.f && dyh >= 0.f)) return true;
    const float a = r1.x, b = r1.y, c = r1.z;
    const float tau = 2.02f * __logf(255.0f * r1.w) + 0.02f;
    const float nb_ia = -b * rcp_approx(a), nb_ic = -b * rcp_approx(c);
    float q = 3.0e38f;
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const float ex_ = k ? dxh : dxl;  // edge dx = ex_: minimise over dy
        const float ty = fminf(fmaxf(nb_ic * ex_, dyl), dyh);
        q = fminf(q, a * ex_ * ex_ + (2.f * b * ex_ + c * ty) * ty);
        const float ey_ = k ? dyh : dyl;  // edge dy = ey_: minimise over dx
        const float tx = fminf(fmaxf(nb_ia * ey_, dxl), dxh);
        q = fminf(q, c * ey_ * ey_ + (2.f * b * ey_ + a * tx) * tx);
    }
    return q <= tau;
}

// ---------------------------------------------------------------- role clocks
// Who waits for whom: compiled with -DF3DGS_ROLE_CLOCKS (tools/time_composite_roles.py; off in the normal build, whose
// SASS is what it is without these lines) every warp of composite_fwd.cu / composite_bwd.cu adds the cycles it spent
// in each mbarrier wait of its role, and in its whole loop, to g_role_clocks of its translation unit.
enum RoleClock {
    kClkProdEmpty, kClkProdLoop,                    // producer: wait for a free stage; whole loop
    kClkAlphaFull, kClkAlphaWempty, kClkAlphaLoop,  // alpha warps: wait for a stage, for a weight slot; whole loop
    kClkFeatWfull, kClkFeatFull, kClkFeatLoop,      // feature warps: wait for a weight slot, for the feature rows
    kRoleClocks
};
#ifdef F3DGS_ROLE_CLOCKS
static __device__ unsigned long long g_role_clocks[kRoleClocks];
// 32-bit cycle counts (a kernel runs far less than 2^32 cycles): the producer has 40 registers
#define ROLE_CLK(...) __VA_ARGS__
#define ROLE_CLK_WAIT(acc, wait)                      \
    do {                                              \
        const uint32_t clk_t_ = (uint32_t)clock64();  \
        wait;                                         \
        acc += (uint32_t)clock64() - clk_t_;          \
    } while (0)
#define ROLE_CLK_ADD(slot, cycles) atomicAdd(&g_role_clocks[slot], (unsigned long long)(cycles))
// g_role_clocks of this translation unit -> out[kRoleClocks]; reset != 0 zeroes them afterwards
#define ROLE_CLK_EXPORT(name)                                                                              \
    extern "C" int name(unsigned long long* out, int reset) {                                              \
        cudaError_t e = cudaMemcpyFromSymbol(out, f3dgs::g_role_clocks, sizeof(f3dgs::g_role_clocks));     \
        const unsigned long long zero[f3dgs::kRoleClocks] = {};                                            \
        if (e == cudaSuccess && reset) e = cudaMemcpyToSymbol(f3dgs::g_role_clocks, zero, sizeof(zero));   \
        return (int)e;                                                                                     \
    }
#else
#define ROLE_CLK(...)
#define ROLE_CLK_WAIT(acc, wait) wait
#endif

// ---------------------------------------------------------------- cp.async (16 bytes per copy, commit groups)
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// wait until at most the N newest commit groups of this thread are pending
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// the same for a warp-uniform run-time count n; n >= kPrefetch - 1 waits for all but the kPrefetch - 1 newest
__device__ __forceinline__ void cp_async_wait_pending(uint32_t n) {
    static_assert(kPrefetch <= 4, "one case per count below kPrefetch - 1");
    if (n >= (uint32_t)kPrefetch - 1u) cp_async_wait<kPrefetch - 1>();
    else if (n == 2) cp_async_wait<2>();
    else if (n == 1) cp_async_wait<1>();
    else cp_async_wait<0>();
}

template <int N>
__device__ __forceinline__ void reg_dec() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void reg_inc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

template <int CH, typename RING>
__device__ __forceinline__ void ring_init(RING& ring, int n_stage_consumers, int n_full_arrivals = 1,
                                          int n_wslot_consumers = 1) {
    // called by all threads before the role split; followed by __syncthreads()
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; s++) {
            mbar_init(&ring.full[s], n_full_arrivals);
            mbar_init(&ring.empty[s], n_stage_consumers);
            mbar_init(&ring.listed[s], 1);
        }
        for (int b = 0; b < RING::kWB; b++)
            for (int j = 0; j < RING::kWJ; j++) {
                mbar_init(&ring.wfull[b][j], 1);
                mbar_init(&ring.wempty[b][j], n_wslot_consumers);
            }
        for (int i = 0; i < kDoneSlots; i++) ring.done_mask[i] = 0;
        mbar_fence_init();
    }
    if (CH > 0) {
        // Zero the rings once per CTA.  A row shorter than CH (C < CH, or the last channel chunk) fills only the head of
        // its stage row; the tail keeps channels of an earlier work item, which the feature warps accumulate too.  Those
        // accumulators never reach memory: the epilogue stores channel ch only if ch < C.
        float4* p = reinterpret_cast<float4*>(&ring.stage[0]);
        const int n16 = (int)(sizeof(ring.stage) / 16);
        for (int i = threadIdx.x; i < n16; i += blockDim.x) p[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        // order these generic-proxy stores before the async-proxy (bulk copy) writes to the same rows
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
}

// Everything the producer needs to know about the view.
struct ProducerArgs {
    const uint2* ranges;
    const uint32_t* point_list;
    const SplatRec* rec;
    const void* features;       // [P, C] of the ring's element type; nullptr: no feature rows (backward, or C == 0)
    const uint32_t* n_contrib;  // backward only: bounds the reverse walk
    int* work_counter;          // zeroed by the launcher; tiles are handed out with atomicAdd
    int W, H, C;
    int tiles_x, num_tiles, chunks;
    int use_bulk;
};

// The producer's view of vp without feature rows (C = 0, one chunk, no bulk copies); the forward adds its feature fields.
inline ProducerArgs producer_args(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                  const SplatRec* rec, const uint32_t* n_contrib, int* work_counter) {
    return ProducerArgs{ranges, point_list, rec, nullptr, n_contrib, work_counter, vp.W, vp.H, 0, (int)vp.grid_x,
                        (int)(vp.grid_x * vp.grid_y), 1, 0};
}

// Channels per work item of the kernels that keep a block's 32 pixels x 4 channels per lane: one of the instantiated
// 32 / 64 / 128; wider features are split into chunks of 128.
inline int channel_chunk(int C) { return C <= 32 ? 32 : (C <= 64 ? 64 : 128); }

// SM count of the current device.  The first call for a device ordinal also opts the kernels K in to `smem` bytes of
// dynamic shared memory: the opt-in is per device (context), so the count is remembered per ordinal and one process
// driving several GPUs works too.  A failed opt-in is returned and retried on the next call; an ordinal of 64 or more
// returns cudaErrorInvalidDevice and leaves `sms` as it is.  With min_ctas > 0 the first call also checks that min_ctas CTAs
// of `threads` threads of every K are resident per SM with that shared memory, and fails with
// cudaErrorLaunchOutOfResources if not: a kernel planned for two CTAs per SM must not silently run at one.
template <auto... K>
cudaError_t device_sms(int& sms, size_t smem, int threads = 0, int min_ctas = 0) {
    static std::atomic<int> sms_of_device[64];  // zero-initialised; set once per device (idempotent)
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    if (sms_of_device[dev].load() == 0) {
        for (const void* k : std::initializer_list<const void*>{reinterpret_cast<const void*>(K)...}) {
            const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
            int ctas = min_ctas;
            if (min_ctas > 0) {
                const cudaError_t eo = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, k, threads, smem);
                if (eo != cudaSuccess) return eo;
            }
            if (ctas < min_ctas) return cudaErrorLaunchOutOfResources;
        }
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sms_of_device[dev].store(n > 0 ? n : 132);
    }
    sms = sms_of_device[dev].load();
    return cudaSuccess;
}

// Producer warp: persistent over work items.  REVERSE: walk each list back to front (backward pass).
// With features (CH > 0) the producer only walks, culls and compacts; it hands each stage's id list to copy_loop() (a
// second warp of the producer group) through `listed[s]`, and that warp issues the stage's bulk copies.  Issuing a bulk
// copy costs the issuing warp ~9 instructions and an R2UR round trip per row (UBLKCP takes uniform registers, so the
// compiler serialises the lanes), a large share of the producer's instructions when a stage's rows are many, and the
// producer is on the pipeline's critical path.
template <int CH, bool REVERSE, typename RING = RingV2<CH>>
__device__ __forceinline__ void producer_loop(RING& ring, const ProducerArgs& pa) {
    using TF = typename RING::Feat;
    constexpr bool COPYWARP = CH > 0;
    const int lane = threadIdx.x & 31;
    int s = 0;
    uint32_t empty_parity = 1;  // fresh barrier: waiting on parity 1 falls through
    ROLE_CLK(uint32_t clk_empty = 0; const uint32_t clk_0 = (uint32_t)clock64();)
    ROLE_CLK_WAIT(clk_empty, mbar_wait(&ring.empty[0], empty_parity));

    uint32_t seq = 0;  // work items this CTA has started
    auto publish = [&](uint32_t n, uint32_t last, uint32_t first, int work) {
        __syncwarp();
        if (lane == 0) {
            Stage<CH, TF>& st = ring.stage[s];
            st.done_slot = seq % kDoneSlots;
            st.n = n;
            st.last = last;
            st.first = first;
            st.work = work;
            mbar_arrive(&ring.full[s]);
            if (COPYWARP) mbar_arrive(&ring.listed[s]);  // release: the stage header, records and ids are visible
        }
        __syncwarp();
    };
    auto advance = [&]() {
        s++;
        if (s == kStages) {
            s = 0;
            empty_parity ^= 1;
        }
        // the producer runs stages ahead: sleep, do not spin
        ROLE_CLK_WAIT(clk_empty, mbar_wait_sleep(&ring.empty[s], empty_parity, 64));
    };

    // ---- the prefetch stream: the record chunks of this CTA's work items, in walk order, copied into ring.rq ahead of
    // their use.  `issued` and `taken` count chunks over the whole kernel; chunk number g lives in slot g % kPrefetch.
    const int num_work = pa.num_tiles * pa.chunks;
    struct Walk {
        int work;               // >= num_work: no more work
        uint32_t begin, count;  // first instance of the tile's list; instances to visit
    };
    auto load_walk = [&](int work) {
        Walk w{work, 0u, 0u};
        if (work < num_work) {
            const int tile = work / pa.chunks;
            const uint2 range = pa.ranges[tile];
            w.begin = range.x;
            w.count = range.y - range.x;
            if (REVERSE) {
                // nothing behind the deepest last-contributor of the tile is ever used
                const int tile_x = tile % pa.tiles_x, tile_y = tile / pa.tiles_x;
                uint32_t tmax = 0;
                const int yy = tile_y * 16 + (lane >> 1), xb = tile_x * 16 + (lane & 1) * 8;
                if (yy < pa.H)
                    for (int i = 0; i < 8; i++)
                        if (xb + i < pa.W) tmax = max(tmax, pa.n_contrib[(size_t)yy * pa.W + xb + i]);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) tmax = max(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
                w.count = min(w.count, tmax);
            }
        }
        return w;
    };
    // i-th visited element of a walk -> index into point_list
    auto list_index = [&](uint32_t begin, uint32_t count, uint32_t i) -> uint32_t {
        return REVERSE ? (begin + count - 1 - i) : (begin + i);
    };

    // Work ids are requested two items ahead (lane 0): `cur` is walked, `nxt` is the item whose first chunks are
    // prefetched while cur's last ones are consumed, and `pending` hides the atomic's round trip.
    int pending = 0;
    Walk cur, nxt;
    {
        int w0 = 0, w1 = 0;
        if (lane == 0) {
            w0 = atomicAdd(pa.work_counter, 1);
            w1 = atomicAdd(pa.work_counter, 1);
            pending = atomicAdd(pa.work_counter, 1);
        }
        cur = load_walk(__shfl_sync(0xffffffffu, w0, 0));
        nxt = load_walk(__shfl_sync(0xffffffffu, w1, 0));
    }
    // Issue cursor: chunk `ic` of the walk (ibegin, icount), which is cur's or, once every chunk of cur is issued, nxt's
    // (in_nxt); id_iss is this lane's Gaussian id of that chunk, loaded one issue ahead of its record copy.  The cursor
    // is exhausted (ic * 32 >= icount) only in nxt: there is no look-ahead beyond the next work item.
    RecQueue& rq = ring.rq;
    uint32_t issued = 0, taken = 0;
    uint32_t ibegin = cur.begin, icount = cur.count, ic = 0, id_iss = 0;
    bool in_nxt = false;
    auto load_id = [&]() -> uint32_t {
        const uint32_t i = ic * 32 + lane;
        return i < icount ? pa.point_list[list_index(ibegin, icount, i)] : 0u;
    };
    auto cursor_cross = [&]() -> bool {  // past cur's last chunk: on to nxt
        if (in_nxt || ic * 32 < icount) return false;
        in_nxt = true;
        ibegin = nxt.begin;
        icount = nxt.count;
        ic = 0;
        return true;
    };
    // Copies the cursor's chunk into slot issued % kPrefetch, one commit group per chunk.  That slot held chunk
    // issued - kPrefetch: wait_group kPrefetch - 1 completes that group before the slot is rewritten, whether the chunk
    // was consumed or dropped by an early exit, so a dropped copy can never land on top of a newer one.
    auto issue = [&]() {
        cp_async_wait<kPrefetch - 1>();
        const uint32_t slot = issued % kPrefetch;
        if (ic * 32 + lane < icount) {
            const float4* r = reinterpret_cast<const float4*>(pa.rec + id_iss);
            cp_async16(&rq.q[slot][0][lane], r);
            cp_async16(&rq.q[slot][1][lane], r + 1);
            cp_async16(&rq.q[slot][2][lane], r + 2);
            rq.id[slot][lane] = id_iss;
        }
        cp_async_commit();
        issued++;
        ic++;
        cursor_cross();
        id_iss = load_id();
    };
    cursor_cross();
    id_iss = load_id();

    for (;;) {
        const int work = cur.work;
        if (work >= num_work) {
            publish(0, 1, 1, -1);
            break;
        }
        const int tile = work / pa.chunks, chunk = work - tile * pa.chunks;
        const int tile_x = tile % pa.tiles_x, tile_y = tile / pa.tiles_x;
        const uint32_t range_begin = cur.begin, walk_count = cur.count;
        const float tx0 = (float)(tile_x * 16), ty0 = (float)(tile_y * 16), tx1 = tx0 + 15.f, ty1 = ty0 + 15.f;
        const int chunk_off = chunk * CH;
        const int row_floats = (CH > 0 && pa.features != nullptr) ? min(CH, pa.C - chunk_off) : 0;
        seq++;
        uint32_t* done = &ring.done_mask[seq % kDoneSlots];
        if (lane == 0) *reinterpret_cast<volatile uint32_t*>(done) = 0;
        __syncwarp();

        auto store_entry = [&](uint32_t slot, uint32_t gid, uint32_t lpos, float4 r0, float4 r1, float4 r2) {
            Stage<CH, TF>& st = ring.stage[s];
            st.rec0[slot] = r0;
            st.rec1[slot] = r1;
            st.rec2[slot] = r2;
            st.listpos[slot] = lpos;
            st.gid[slot] = gid;
            if (CH > 0 && row_floats > 0) {
                const TF* src = static_cast<const TF*>(pa.features) + (size_t)gid * pa.C + chunk_off;
                if (!pa.use_bulk)  // unaligned rows or rows not a multiple of 16 bytes: the producer loads the row
                    for (int c = 0; c < row_floats; c++) st.feat[slot][c] = __ldg(src + c);
            }
        };

        uint32_t fill = 0, first = 1;
        const uint32_t nchunks = (walk_count + 31) / 32;
        for (uint32_t c = 0; c < nchunks; c++) {
            if (*reinterpret_cast<volatile uint32_t*>(done) == (1u << kBlocksPerTile) - 1u) {
                // Early exit: the issued chunks of this walk are dropped by stepping `taken` over them, and the cursor
                // moves on to nxt.  Their copies may still be in flight; the slot sequence keeps running, and issue()
                // waits for a slot's previous group before it rewrites the slot.
                taken += (in_nxt ? nchunks : ic) - c;
                if (!in_nxt) {
                    ic = nchunks;
                    cursor_cross();
                    id_iss = load_id();
                }
                break;
            }
            // this chunk and kPrefetch - 1 chunks behind it in flight, across the boundary to the next work item
            while (issued - taken < (uint32_t)kPrefetch && ic * 32 < icount) issue();
            cp_async_wait_pending(issued - taken - 1);  // groups newer than this chunk's may still be in flight
            __syncwarp();
            const uint32_t qs = taken % kPrefetch;
            taken++;
            // every lane reads back what it copied itself: conflict-free LDS.128
            const float4 a0 = rq.q[qs][0][lane], a1 = rq.q[qs][1][lane], a2 = rq.q[qs][2][lane];
            const uint32_t id_cur = rq.id[qs][lane];

            const uint32_t i0 = c * 32 + lane;
            const bool valid = i0 < walk_count;
            // does the alpha >= 1/255 footprint reach this tile?  (conservative, see alpha_extent)
            const bool keep = valid && footprint_hits_rect(a0, a1, tx0, tx1, ty0, ty1);
            const uint32_t m = __ballot_sync(0xffffffffu, keep);
            const uint32_t cnt = __popc(m);
            const uint32_t rank = __popc(m & ((1u << lane) - 1u));
            const uint32_t lpos = list_index(range_begin, walk_count, i0) - range_begin + 1;
            const uint32_t room = kStageEntries - fill;
            if (keep && rank < room) store_entry(fill + rank, id_cur, lpos, a0, a1, a2);
            if (cnt >= room) {
                publish(kStageEntries, 0, first, work);
                first = 0;
                advance();
                if (keep && rank >= room) store_entry(rank - room, id_cur, lpos, a0, a1, a2);
                fill = cnt - room;
            } else {
                fill += cnt;
            }
        }
        publish(fill, 1, first, work);
        advance();

        // next work item.  Every chunk of cur was issued or stepped over, so the cursor is in nxt.
        const int new_work = __shfl_sync(0xffffffffu, pending, 0);
        if (lane == 0 && new_work < num_work) pending = atomicAdd(pa.work_counter, 1);
        cur = nxt;
        nxt = load_walk(new_work);
        in_nxt = false;
        if (cursor_cross()) id_iss = load_id();
    }
    cp_async_wait<0>();  // dropped copies land before the warp retires
    ROLE_CLK(if (lane == 0) {
        ROLE_CLK_ADD(kClkProdEmpty, clk_empty);
        ROLE_CLK_ADD(kClkProdLoop, (uint32_t)clock64() - clk_0);
    })
}

// Second warp of the producer group (forward with features): fetches the feature rows of each listed stage.
template <int CH, typename TF>
__device__ __forceinline__ void copy_loop(RingV2<CH, TF>& ring, const ProducerArgs& pa) {
    const int lane = threadIdx.x & 31;
    int s = 0;
    uint32_t parity = 0;
    for (;;) {
        mbar_wait(&ring.listed[s], parity);
        Stage<CH, TF>& st = ring.stage[s];
        const uint32_t n = st.n;
        const int work = st.work;
        if (work < 0) {
            if (lane == 0) mbar_arrive(&ring.full[s]);
            break;
        }
        const int chunk_off = (work % pa.chunks) * CH;
        const uint32_t row_bytes = (uint32_t)min(CH, pa.C - chunk_off) * (uint32_t)sizeof(TF);
        if (pa.use_bulk && n > 0) {
            if (lane == 0) mbar_arrive_expect_tx(&ring.full[s], n * row_bytes);
            __syncwarp();
            if (lane < n)
                bulk_g2s(&st.feat[lane][0],
                         static_cast<const TF*>(pa.features) + (size_t)st.gid[lane] * pa.C + chunk_off, row_bytes,
                         &ring.full[s]);
        } else {
            if (lane == 0) mbar_arrive(&ring.full[s]);
        }
        if (++s == kStages) {
            s = 0;
            parity ^= 1;
        }
    }
}

}  // namespace f3dgs
