// Shared machinery of the forward and backward composite kernels (persistent, warp-specialised).
//
// The reference renders one 16x16 tile per 256-thread block, every thread doing everything
// (forward.cu:261-396).  Here a persistent CTA pulls tiles from an atomic counter and splits the
// work over warp roles that talk only through shared-memory rings + mbarriers:
//
//   producer group (4)    warp 0 walks the tile's slice of the depth-sorted instance list, drops the
//                         instances whose alpha >= 1/255 footprint cannot reach the tile, and fills
//                         a ring of stages with 48-byte splat records via 128-bit loads.  When there
//                         are features, warp 1 (the copy warp) fetches the stage's C-wide feature
//                         rows with 1-D TMA bulk copies (cp.async.bulk -> UBLKCP) that complete on
//                         the stage's `full` mbarrier.  The producer runs ahead across tile
//                         boundaries, so the next tile's first stage is already resident when the
//                         consumers get there (no per-tile start-up bubble).  Warps 2 and 3 retire.
//   alpha warps (8)       warp a owns the 8x4 pixel block a of the tile, one pixel per lane: alpha,
//                         the T recurrence, RGB/depth (and in the backward every geometric gradient
//                         term).  In the forward they publish the blend weights w = alpha*T as a
//                         [instance][pixel] tile plus a per-instance pixel mask in a small per-block
//                         ring (`wfull`/`wempty`).
//   feature warps (8)     forward only: warp b consumes block b's weight tiles with one float4 of
//                         channels per lane; all 32 pixels x 4 channels of the block stay in
//                         registers, and the weights arrive as broadcast LDS.128 per 2x2 pixel quad.
//
// The forward launches all 20 warps (composite_fwd.cu); the backward geometry kernel launches the
// producer group and the alpha warps only (composite_bwd.cu).
#pragma once
#include "kernels.h"

namespace f3dgs {

constexpr int kBlocksPerTile = 8;   // 8x4-pixel blocks in a 16x16 tile
constexpr int kProducerWarp = 0;    // warps 0..3: producer warpgroup
constexpr int kAlphaWarp0 = 4;      // then one alpha warp per pixel block
constexpr int kAlphaWarps = kBlocksPerTile;
constexpr int kFeatWarp0 = kAlphaWarp0 + kAlphaWarps;  // then one feature warp per pixel block (forward)
constexpr int kRegsProducer = 40;   // setmaxnreg of the producer group
constexpr int kStageEntries = 32;
constexpr int kStages = 6;
constexpr int kWSlots = 2;
constexpr int kDoneSlots = 8;       // > kStages: the producer is never further ahead than that.  Slots are indexed by the
                                    // CTA's own work sequence number, NOT by the work id: ids come from a global
                                    // atomic counter, so two items in flight in one CTA can be congruent mod 8.

template <int CH>
struct alignas(128) Stage {
    float feat[CH > 0 ? kStageEntries : 1][CH > 0 ? CH : 4];  // CH == 0: 16 B dummy, never touched
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
    uint32_t km;                   // which instances have pm != 0
    uint32_t last;
    uint32_t first;
    int32_t work;
};

template <int CH>
struct alignas(128) RingV2 {
    static constexpr int kWB = kBlocksPerTile, kWJ = kWSlots;  // dimensions of the weight-slot ring
    Stage<CH> stage[kStages];
    WSlot ws[kBlocksPerTile][kWSlots];
    uint64_t full[kStages];
    uint64_t empty[kStages];
    uint64_t listed[kStages];  // records + ids of the stage are written: the copy warp may fetch its feature rows
    uint64_t wfull[kBlocksPerTile][kWSlots];
    uint64_t wempty[kBlocksPerTile][kWSlots];
    uint32_t done_mask[kDoneSlots];  // bit b set: pixel block b of that work item needs no more instances
};

// The same ring without feature rows or weight slots, for the backward geometry kernel, which has no feature warps:
// 14 KB instead of 83 KB of shared memory, so that two CTAs fit on an SM.  The one-element `ws` / `wfull` / `wempty` are
// not used; ring_init<> initialises the two barriers.
struct alignas(128) RingSlim {
    static constexpr int kWB = 1, kWJ = 1;
    Stage<0> stage[kStages];
    WSlot ws[1][1];
    uint64_t full[kStages];
    uint64_t empty[kStages];
    uint64_t listed[kStages];
    uint64_t wfull[1][1];
    uint64_t wempty[1][1];
    uint32_t done_mask[kDoneSlots];
};

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

// pixel <-> lane mapping inside a block: 2x2 quads, quad q = lane>>2 laid out 4 across
__device__ __forceinline__ int lane_px(int lane) { return ((lane >> 2) & 3) * 2 + (lane & 1); }
__device__ __forceinline__ int lane_py(int lane) { return (lane >> 4) * 2 + ((lane >> 1) & 1); }

template <int N>
__device__ __forceinline__ void reg_dec() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void reg_inc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

template <int CH, typename RING>
__device__ __forceinline__ void ring_init(RING& ring, int n_stage_consumers, int n_full_arrivals = 1) {
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
                mbar_init(&ring.wempty[b][j], 1);
            }
        for (int i = 0; i < kDoneSlots; i++) ring.done_mask[i] = 0;
        mbar_fence_init();
    }
    if (CH > 0) {
        // Zero the rings once per CTA.  A row shorter than CH (C < CH, or the last channel chunk) fills only the head of
        // its stage row; the tail keeps channels of an earlier work item, which the feature warps accumulate too.  Those
        // accumulators never reach memory: the epilogue stores channel ch only if ch < C.
        float4* p = reinterpret_cast<float4*>(&ring.stage[0]);
        const int n16 = (int)(sizeof(Stage<CH>) * kStages / 16);
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
    const float* features;      // nullptr: no feature rows (backward, or C == 0)
    const uint32_t* n_contrib;  // backward only: bounds the reverse walk
    int* work_counter;          // zeroed by the launcher; tiles are handed out with atomicAdd
    int W, H, C;
    int tiles_x, num_tiles, chunks;
    int use_bulk;
};

// Producer warp: persistent over work items.  REVERSE: walk each list back to front (backward pass).
// With features (CH > 0) the producer only walks, culls and compacts; it hands each stage's id list to copy_loop() (a
// second warp of the producer group) through `listed[s]`, and that warp issues the stage's bulk copies.  Issuing a bulk
// copy costs the issuing warp ~9 instructions and an R2UR round trip per row (UBLKCP takes uniform registers, so the
// compiler serialises the lanes), a large share of the producer's instructions when a stage's rows are many, and the
// producer is on the pipeline's critical path.
template <int CH, bool REVERSE, typename RING = RingV2<CH>>
__device__ __forceinline__ void producer_loop(RING& ring, const ProducerArgs& pa) {
    constexpr bool COPYWARP = CH > 0;
    const int lane = threadIdx.x & 31;
    int s = 0;
    uint32_t empty_parity = 1;  // fresh barrier: waiting on parity 1 falls through
    mbar_wait(&ring.empty[0], empty_parity);

    uint32_t seq = 0;  // work items this CTA has started
    auto publish = [&](uint32_t n, uint32_t last, uint32_t first, int work) {
        __syncwarp();
        if (lane == 0) {
            Stage<CH>& st = ring.stage[s];
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
        mbar_wait_sleep(&ring.empty[s], empty_parity, 64);  // the producer runs stages ahead: sleep, do not spin
    };

    const int num_work = pa.num_tiles * pa.chunks;
    int pending = 0;  // lane 0: the next work item, requested one item ahead so the atomic's round trip is hidden
    if (lane == 0) pending = atomicAdd(pa.work_counter, 1);
    for (;;) {
        const int work = __shfl_sync(0xffffffffu, pending, 0);
        if (lane == 0 && work < num_work) pending = atomicAdd(pa.work_counter, 1);
        if (work >= num_work) {
            publish(0, 1, 1, -1);
            break;
        }
        const int tile = work / pa.chunks, chunk = work - tile * pa.chunks;
        const int tile_x = tile % pa.tiles_x, tile_y = tile / pa.tiles_x;
        const uint2 range = pa.ranges[tile];
        const uint32_t range_begin = range.x;
        uint32_t walk_count = range.y - range.x;
        if (REVERSE) {
            // nothing behind the deepest last-contributor of the tile is ever used
            uint32_t tmax = 0;
            const int yy = tile_y * 16 + (lane >> 1), xb = tile_x * 16 + (lane & 1) * 8;
            if (yy < pa.H)
                for (int i = 0; i < 8; i++)
                    if (xb + i < pa.W) tmax = max(tmax, pa.n_contrib[(size_t)yy * pa.W + xb + i]);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) tmax = max(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
            walk_count = min(walk_count, tmax);
        }
        const float tx0 = (float)(tile_x * 16), ty0 = (float)(tile_y * 16), tx1 = tx0 + 15.f, ty1 = ty0 + 15.f;
        const int chunk_off = chunk * CH;
        const int row_floats = (CH > 0 && pa.features != nullptr) ? min(CH, pa.C - chunk_off) : 0;
        seq++;
        uint32_t* done = &ring.done_mask[seq % kDoneSlots];
        if (lane == 0) *reinterpret_cast<volatile uint32_t*>(done) = 0;
        __syncwarp();

        auto list_index = [&](uint32_t i) -> uint32_t {  // i-th visited element -> index into point_list
            return REVERSE ? (range_begin + walk_count - 1 - i) : (range_begin + i);
        };
        auto store_entry = [&](uint32_t slot, uint32_t gid, uint32_t lpos, float4 r0, float4 r1, float4 r2) {
            Stage<CH>& st = ring.stage[s];
            st.rec0[slot] = r0;
            st.rec1[slot] = r1;
            st.rec2[slot] = r2;
            st.listpos[slot] = lpos;
            st.gid[slot] = gid;
            if (CH > 0 && row_floats > 0) {
                const float* src = pa.features + (size_t)gid * pa.C + chunk_off;
                if (!pa.use_bulk)  // unaligned rows or C % 4 != 0: no bulk copies, the producer loads the row
                    for (int c = 0; c < row_floats; c++) st.feat[slot][c] = __ldg(src + c);
            }
        };

        uint32_t fill = 0, first = 1;
        // two-deep software pipeline on the dependent loads (list index -> id -> record)
        const uint32_t nchunks = (walk_count + 31) / 32;
        uint32_t id_cur = 0, id_nxt = 0;
        float4 a0, a1, a2;
        a0 = a1 = a2 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (nchunks > 0) {
            if (lane < walk_count) id_cur = pa.point_list[list_index(lane)];
            if (32 + lane < walk_count) id_nxt = pa.point_list[list_index(32 + lane)];
            if (lane < walk_count) {
                const float4* r = reinterpret_cast<const float4*>(pa.rec + id_cur);
                a0 = __ldg(r); a1 = __ldg(r + 1); a2 = __ldg(r + 2);
            }
        }
        for (uint32_t c = 0; c < nchunks; c++) {
            if (*reinterpret_cast<volatile uint32_t*>(done) == (1u << kBlocksPerTile) - 1u) break;
            float4 b0, b1, b2;
            b0 = b1 = b2 = make_float4(0.f, 0.f, 0.f, 0.f);
            const uint32_t i1 = (c + 1) * 32 + lane, i2 = (c + 2) * 32 + lane;
            uint32_t id_nn = 0;
            if (i1 < walk_count) {
                const float4* r = reinterpret_cast<const float4*>(pa.rec + id_nxt);
                b0 = __ldg(r); b1 = __ldg(r + 1); b2 = __ldg(r + 2);
            }
            if (i2 < walk_count) id_nn = pa.point_list[list_index(i2)];

            const uint32_t i0 = c * 32 + lane;
            const bool valid = i0 < walk_count;
            // does the alpha >= 1/255 footprint reach this tile?  (conservative, see alpha_extent)
            const bool keep = valid && footprint_hits_rect(a0, a1, tx0, tx1, ty0, ty1);
            const uint32_t m = __ballot_sync(0xffffffffu, keep);
            const uint32_t cnt = __popc(m);
            const uint32_t rank = __popc(m & ((1u << lane) - 1u));
            const uint32_t lpos = list_index(i0) - range_begin + 1;
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
            a0 = b0; a1 = b1; a2 = b2;
            id_cur = id_nxt;
            id_nxt = id_nn;
        }
        publish(fill, 1, first, work);
        advance();
    }
}

// Second warp of the producer group (forward with features): fetches the feature rows of each listed stage.
template <int CH>
__device__ __forceinline__ void copy_loop(RingV2<CH>& ring, const ProducerArgs& pa) {
    const int lane = threadIdx.x & 31;
    int s = 0;
    uint32_t parity = 0;
    for (;;) {
        mbar_wait(&ring.listed[s], parity);
        Stage<CH>& st = ring.stage[s];
        const uint32_t n = st.n;
        const int work = st.work;
        if (work < 0) {
            if (lane == 0) mbar_arrive(&ring.full[s]);
            break;
        }
        const int chunk_off = (work % pa.chunks) * CH;
        const uint32_t row_bytes = (uint32_t)min(CH, pa.C - chunk_off) * 4u;
        if (pa.use_bulk && n > 0) {
            if (lane == 0) mbar_arrive_expect_tx(&ring.full[s], n * row_bytes);
            __syncwarp();
            if (lane < n)
                bulk_g2s(&st.feat[lane][0], pa.features + (size_t)st.gid[lane] * pa.C + chunk_off, row_bytes,
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
