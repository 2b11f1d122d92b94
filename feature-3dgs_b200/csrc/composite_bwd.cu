// Backward tile composite: walks each tile's instance list back to front and produces the
// per-Gaussian gradients of colour, feature, depth, opacity, conic and 2-D mean.
// Reference: backward.cu:407-620 (renderCUDA<3>), semantics restated in SURVEY.md A.5 / D.1.
//
// The reference issues (C+10) same-address global atomics per blended (pixel, Gaussian) pair.
// Here (roles as in composite_common.cuh, persistent over tiles):
//   alpha warp a   lane = pixel of blocks 2a / 2a+1: recomputes alpha, unwinds T, and forms the 10 scalar
//       gradient terms of the pair (2-D mean x2, conic x3, opacity, depth, colour x3).  Lanes park
//       their terms in a [value][instance slot][pixel] shared tile; when 8 instances are parked the
//       tile is summed row-wise (one lane per row, conflict-free padded rows) and each row sum
//       becomes ONE red.global.add -> 32x fewer atomics, none contended inside the warp.  It also
//       publishes w = alpha*T and the pixel masks to the block's feature warp.
//   feature warp b lane = float4 of channels: keeps dL/dfeature_map of all 32 pixels x 4 channels
//       in registers for the whole tile (the upstream gradient is read from HBM exactly once);
//       per blended instance  g[4] = sum_pixels w[pixel] * dO[pixel][4]  is 2x2-quad sparse FMAs
//       fed by broadcast LDS.128 of the weights, then one red.global.add.v4.f32 per lane: a fully
//       coalesced 512-byte vector reduction per (block, instance) at C = 128.
// As in the reference, the feature loss does not feed dL/dalpha (backward.cu:575 is disabled).
// No features are read at all: the feature gradient needs only w = alpha*T and dL/dout.
#include <cstdio>
#include <cstdlib>

#include "composite_common.cuh"

namespace f3dgs {

#ifndef F3DGS_TIMING_BUILD
#define F3DGS_TIMING_BUILD 0   // build.py sets 1 when env F3DGS_TIMING_BUILD=1: per-role cycle counters (see composite_fwd.cu)
#endif
// Diagnostic builds only (WRONG RESULTS, timing experiments): drop the feature-gradient / geometric-gradient global reductions
// to measure what the red.global.add traffic costs (tools/run_r1e.sh).
#ifndef F3DGS_DIAG_NO_FEAT_RED
#define F3DGS_DIAG_NO_FEAT_RED 0
#endif
#ifndef F3DGS_DIAG_NO_FMA
#define F3DGS_DIAG_NO_FMA 0   // feature warps consume their slots without FMAs or reductions (alpha-limited time)
#endif
#ifndef F3DGS_DIAG_NO_GEOM_RED
#define F3DGS_DIAG_NO_GEOM_RED 0
#endif
static constexpr bool kTimingB = F3DGS_TIMING_BUILD != 0;
#define BTICK() ((kTimingB && args.dbg) ? clock64() : 0ll)

#ifndef F3DGS_PAIR_SKIP
#define F3DGS_PAIR_SKIP 1   // 1 (with F3DGS_FFMA2): skip the paired FMAs of a quad row whose two pixels did not blend
#endif
#ifndef F3DGS_FFMA2
#define F3DGS_FFMA2 1   // 1: feature-gradient loop on paired accumulators (fma2_rn), see composite_fwd.cu
#endif

#ifndef F3DGS_RED_SLOTS
#define F3DGS_RED_SLOTS 8
#endif
#ifndef F3DGS_SLIM_CTAS
#define F3DGS_SLIM_CTAS 2   // CTAs per SM of the alpha-only (SLIM) layout
#endif
constexpr int kRedSlots = F3DGS_RED_SLOTS;
constexpr int kSlimCtas = F3DGS_SLIM_CTAS;
constexpr int kRedVals = 10;
constexpr int kRedRows = kRedSlots * kRedVals;
constexpr int kRedStride = 36;  // floats per row: lanes park at [row][lane] (conflict-free), rows are summed with
                                // LDS.128 (quarter-warp wavefronts: rows r..r+7 start 4 banks apart -> conflict-free)

// Backward register budget for the 20-warp layout (640 threads x 96 = 61440 registers in the CTA pool):
// 4x32x40 + 8x32xA + 8x32xF <= 61440  =>  A + F <= 220.  Default 64 / 152; -DF3DGS_BWD_A1=72 -DF3DGS_BWD_F1=144 trades
// feature-warp headroom for fewer spills in the alpha warps (experiment).
#ifndef F3DGS_BWD_A1
#define F3DGS_BWD_A1 64
#define F3DGS_BWD_F1 152
#endif
template <int BPA>
struct BwdLayout : Layout<BPA> {
    static constexpr int kRegsAlpha = BPA == 2 ? 104 : F3DGS_BWD_A1;
    static constexpr int kRegsFeature = BPA == 2 ? 184 : F3DGS_BWD_F1;
};

template <typename RING>
struct alignas(128) BwdSmemT {
    RING ring;
    float red[kBlocksPerTile][kRedRows][kRedStride];
    uint32_t red_gid[kBlocksPerTile][kRedSlots];
};
using BwdSmem = BwdSmemT<RingV2<0>>;

struct BwdArgs {
    ProducerArgs pa;
    const float* bg;
    const float* final_T;
    const uint32_t* n_contrib;
    const float* dL_dpix;
    const float* dL_dfeat_pix;
    const float* dL_ddepth;
    float* dL_dmean2D;   // [P,3]
    float* dL_dconic;    // [P,4]
    float* dL_dopacity;  // [P]
    float* dL_dcolor;    // [P,3]
    float* dL_dfeature;  // [P,C]
    float* dL_dz;        // [P]
    int vec_io;          // bit0: 128-bit loads of dL_dfeat_pix, bit1: red.v4 into dL_dfeature
    long long* dbg;      // F3DGS_TIMING=1 (timing builds only): per-warp cycle counters [cta][warp][8], else nullptr
    // EMIT kernels (two-kernel backward): per (tile, 8x4 block) lists of the instances that blended in the block
    float* list_w;        // [8R][32] blend weights w = alpha * T (the backward's unwound T), entry (8*range.x + b*len + i)
    uint2* list_meta;     // [8R]     {Gaussian id, pixel mask}
    uint32_t* list_cnt;   // [8T]     entries written per (tile, block)
};

// destination of reduced value v (0..9) of Gaussian gid: reference backward.cu:560-610 (atomicAdd targets)
__device__ __forceinline__ float* geom_dst(const BwdArgs& args, int v, uint32_t gid) {
    switch (v) {
        case 0: return args.dL_dmean2D + 3 * (size_t)gid;
        case 1: return args.dL_dmean2D + 3 * (size_t)gid + 1;
        case 2: return args.dL_dconic + 4 * (size_t)gid;
        case 3: return args.dL_dconic + 4 * (size_t)gid + 1;
        case 4: return args.dL_dconic + 4 * (size_t)gid + 3;
        case 5: return args.dL_dopacity + gid;
        case 6: return args.dL_dz + gid;
        default: return args.dL_dcolor + 3 * (size_t)gid + (v - 7);
    }
}


// SLIM (geometric pass of the two-pass mode, CH == 0): 12 warps, ring without weight slots (106 KB of shared memory instead
// of 175 KB), two CTAs per SM; the alpha warps keep the launch register count (80) instead of shrinking to 64.
template <int CH, int BPA, bool SLIM = false, bool EMIT = false>
__global__ void __launch_bounds__(SLIM ? (kAlphaWarp0 + Layout<BPA>::kAlphaWarps) * 32 : Layout<BPA>::kThreads, SLIM ? kSlimCtas : 1)
composite_bwd_kernel(const BwdArgs args) {
    static_assert(!SLIM || CH == 0, "the slim layout has no feature warps");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using RING = typename RingSelect<0, SLIM>::type;
    using SMEM = BwdSmemT<RING>;
    SMEM& sm = *reinterpret_cast<SMEM*>(smem_raw);
    RING& ring = sm.ring;
    // The warp index goes through a shuffle so that ptxas knows it is warp-uniform: role branches, ring/slot addresses
    // and everything loaded from them (instance masks, work ids) then live in uniform registers, the per-quad branches
    // of the feature loop need no BSSY/BSYNC reconvergence pair, and nothing is re-derived from SR_TID inside the loops.
    const int warp = F3DGS_UNIFORM_WARP ? __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0) : (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int W = args.pa.W, H = args.pa.H, C = args.pa.C;
    const size_t HW = (size_t)H * W;

    using L = BwdLayout<BPA>;
    ring_init<0>(ring, CH > 0 ? L::kAlphaWarps + kBlocksPerTile : L::kAlphaWarps, CH > 0);
    __syncthreads();

    // ======================================================================== producer group
    if (warp < kAlphaWarp0) {
        reg_dec<L::kRegsProducer>();
        if (warp == kProducerWarp) producer_loop<0, true, false, RING>(ring, args.pa);
        return;
    }

    // ======================================================================== alpha warps
    if (warp < L::kFeatWarp0) {
        if (!SLIM) reg_dec<L::kRegsAlpha>();
        const int a = warp - kAlphaWarp0;  // owns blocks BPA*a .. BPA*a + BPA-1
        float(*red)[kRedStride] = sm.red[a];
        uint32_t* red_gid = sm.red_gid[a];
        uint32_t nslots = 0;  // warp-uniform; rows of both blocks share the scratch
        int s = 0, j = 0;
        uint32_t parity = 0, wparity = 1;
        struct Px {
            float T, T_final, pxf, pyf, fbx0, fby0, dLp0, dLp1, dLp2, dLd, bg_dot;
            float ar0, ar1, ar2, lc0, lc1, lc2, last_alpha, accum_depth, last_depth;
            uint32_t last_contrib, wmax;
            bool inside;
        } P[BPA];
#pragma unroll
        for (int bi = 0; bi < BPA; bi++) {
            P[bi] = Px{};
        }
        bool do_geom = false;
        size_t ebase[BPA];      // EMIT: first list entry of this (tile, block)
        uint32_t ecount[BPA];   // EMIT: entries written so far
        int etile = 0;
#pragma unroll
        for (int bi = 0; bi < BPA; bi++) { ebase[bi] = 0; ecount[bi] = 0; }
        const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;
        long long tA_full = 0, tA_wempty = 0, tA_flush = 0, nA_hits = 0, nA_pm = 0;
        const long long tA_total = BTICK();

        auto flush = [&]() {
            const long long tf_ = BTICK();
            __syncwarp();
            for (int r = lane; r < kRedRows; r += 32) {
                const int slot = r % kRedSlots, v = r / kRedSlots;
                if (slot < (int)nslots) {
                    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
                    const float4* row = reinterpret_cast<const float4*>(red[r]);
#pragma unroll
                    for (int jj = 0; jj < 8; jj++) {
                        const float4 q = row[jj];
                        s0 += q.x;
                        s1 += q.y;
                        s2 += q.z;
                        s3 += q.w;
                    }
                    const float sum = (s0 + s1) + (s2 + s3);
                    const uint32_t gid = red_gid[slot];
                    float* dst;
                    switch (v) {
                        case 0: dst = args.dL_dmean2D + 3 * (size_t)gid; break;
                        case 1: dst = args.dL_dmean2D + 3 * (size_t)gid + 1; break;
                        case 2: dst = args.dL_dconic + 4 * (size_t)gid; break;
                        case 3: dst = args.dL_dconic + 4 * (size_t)gid + 1; break;
                        case 4: dst = args.dL_dconic + 4 * (size_t)gid + 3; break;
                        case 5: dst = args.dL_dopacity + gid; break;
                        case 6: dst = args.dL_dz + gid; break;
                        default: dst = args.dL_dcolor + 3 * (size_t)gid + (v - 7); break;
                    }
                    if (!F3DGS_DIAG_NO_GEOM_RED) red_add_f1(dst, sum);
                    else if (sum == 123456.789f) red_add_f1(dst, sum);  // keeps the row sums alive
                }
            }
            __syncwarp();
            nslots = 0;
            tA_flush += BTICK() - tf_;
        };

        for (;;) {
            { const long long t_ = BTICK(); mbar_wait(&ring.full[s], parity); tA_full += BTICK() - t_; }
            Stage<0>& st = ring.stage[s];
            const uint32_t n = st.n, last = st.last, first = st.first;
            const int work = st.work;
            if (work < 0) break;
            if (first) {
                const int tile = work / args.pa.chunks, chunk = work - tile * args.pa.chunks;
                const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
                do_geom = (chunk == 0);
                if (EMIT) {
                    etile = tile;
                    const uint2 rg = args.pa.ranges[tile];
#pragma unroll
                    for (int bi = 0; bi < BPA; bi++) {
                        ebase[bi] = 8 * (size_t)rg.x + (size_t)(BPA * a + bi) * (rg.y - rg.x);
                        ecount[bi] = 0;
                    }
                }
#pragma unroll
                for (int bi = 0; bi < BPA; bi++) {
                    const int b = BPA * a + bi;
                    Px& p = P[bi];
                    const int bx0 = tile_x * 16 + (b & 1) * 8, by0 = tile_y * 16 + (b >> 1) * 4;
                    const int px = bx0 + lane_px(lane), py = by0 + lane_py(lane);
                    p.inside = px < W && py < H;
                    p.pxf = (float)px; p.pyf = (float)py; p.fbx0 = (float)bx0; p.fby0 = (float)by0;
                    const size_t pix = p.inside ? (size_t)py * W + px : 0;
                    p.T_final = p.inside ? args.final_T[pix] : 0.f;
                    p.T = p.T_final;
                    p.last_contrib = p.inside ? args.n_contrib[pix] : 0u;
                    p.dLp0 = p.dLp1 = p.dLp2 = p.dLd = 0.f;
                    if (p.inside) {
                        p.dLp0 = args.dL_dpix[pix];
                        p.dLp1 = args.dL_dpix[HW + pix];
                        p.dLp2 = args.dL_dpix[2 * HW + pix];
                        p.dLd = args.dL_ddepth[pix];
                    }
                    p.bg_dot = args.bg[0] * p.dLp0 + args.bg[1] * p.dLp1 + args.bg[2] * p.dLp2;
                    p.ar0 = p.ar1 = p.ar2 = p.lc0 = p.lc1 = p.lc2 = 0.f;
                    p.last_alpha = p.accum_depth = p.last_depth = 0.f;
                    uint32_t wm = p.last_contrib;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) wm = max(wm, __shfl_xor_sync(0xffffffffu, wm, o));
                    p.wmax = wm;
                }
            }
#pragma unroll
            for (int bi = 0; bi < BPA; bi++) {
                const int b = BPA * a + bi;
                Px& p = P[bi];
                WSlot* ws = &ring.ws[b][j];
                if (CH > 0) { const long long t_ = BTICK(); mbar_wait(&ring.wempty[b][j], wparity); tA_wempty += BTICK() - t_; }
                uint32_t km = 0;
                if (n > 0 && p.wmax > 0) {
                    bool hit = false;
                    if (lane < n) {
#if F3DGS_EXACT_CULL
                        hit = (st.listpos[lane] <= p.wmax) &&
                              footprint_hits_rect(st.rec0[lane], st.rec1[lane], p.fbx0, p.fbx0 + 7.f, p.fby0, p.fby0 + 3.f);
#else
                        const float4 r0 = st.rec0[lane];
                        hit = (st.listpos[lane] <= p.wmax) && (r0.x + r0.z >= p.fbx0) && (r0.x - r0.z <= p.fbx0 + 7.f) &&
                              (r0.y + r0.w >= p.fby0) && (r0.y - r0.w <= p.fby0 + 3.f);
#endif
                    }
                    uint32_t am = __ballot_sync(0xffffffffu, hit);
                    if (kTimingB) nA_hits += __popc(am);
                    while (am) {
                        // branch-free evaluation of two instances per trip (see composite_fwd.cu)
                        int kk[2];
                        bool vk[2];
                        float al[2], Gv[2], dxv[2], dyv[2];
#pragma unroll
                        for (int u = 0; u < 2; u++) {
                            vk[u] = am != 0;
                            kk[u] = vk[u] ? (__ffs(am) - 1) : 0;
                            am &= am - 1;
                        }
#pragma unroll
                        for (int u = 0; u < 2; u++) {
                            const float4 r0 = st.rec0[kk[u]];
                            const float4 r1 = st.rec1[kk[u]];
                            // same expression trees as reference backward.cu:525-535
                            const float dx = r0.x - p.pxf, dy = r0.y - p.pyf;
                            const float power = -0.5f * (r1.x * dx * dx + r1.z * dy * dy) - r1.y * dx * dy;
                            const float Gs = expf(power);
                            const float av = fminf(0.99f, r1.w * Gs);
                            al[u] = (vk[u] && !(power > 0.0f) && !(av < 1.0f / 255.0f)) ? av : 0.f;
                            Gv[u] = Gs; dxv[u] = dx; dyv[u] = dy;
                        }
#pragma unroll
                        for (int u = 0; u < 2; u++) {
                            if (!vk[u]) break;  // warp-uniform, only in the last trip
                            const int k = kk[u];
                            const float alpha = al[u];
                            const bool contrib = p.inside && alpha > 0.f && st.listpos[k] <= p.last_contrib;
                            float wgt = 0.f;
                            float v[kRedVals];
#pragma unroll
                            for (int i = 0; i < kRedVals; i++) v[i] = 0.f;
                            if (contrib) {
                                const float4 r1 = st.rec1[k];
                                const float4 r2 = st.rec2[k];
                                // 1/(1-alpha), 1-alpha in [0.01, 1]: one MUFU.RCP (<= 1 ulp) serves both the T unwind and
                                // the background term, where the reference divides twice (backward.cu:541,583); the
                                // unwound T differs from the reference's by a few ulp after a whole tile list.
                                const float inv_1ma = rcp_approx(1.f - alpha);
                                p.T = p.T * inv_1ma;
                                wgt = alpha * p.T;
                                float dL_dalpha;
                                p.ar0 = p.last_alpha * p.lc0 + (1.f - p.last_alpha) * p.ar0; p.lc0 = r2.x;
                                p.ar1 = p.last_alpha * p.lc1 + (1.f - p.last_alpha) * p.ar1; p.lc1 = r2.y;
                                p.ar2 = p.last_alpha * p.lc2 + (1.f - p.last_alpha) * p.ar2; p.lc2 = r2.z;
                                dL_dalpha = (r2.x - p.ar0) * p.dLp0 + (r2.y - p.ar1) * p.dLp1 + (r2.z - p.ar2) * p.dLp2;
                                v[7] = wgt * p.dLp0; v[8] = wgt * p.dLp1; v[9] = wgt * p.dLp2;
                                p.accum_depth = p.last_alpha * p.last_depth + (1.f - p.last_alpha) * p.accum_depth;
                                p.last_depth = r2.w;
                                dL_dalpha += (r2.w - p.accum_depth) * p.dLd;
                                dL_dalpha *= p.T;
                                p.last_alpha = alpha;
                                dL_dalpha += (-p.T_final * inv_1ma) * p.bg_dot;
                                const float Gs = Gv[u], dx = dxv[u], dy = dyv[u];
                                const float dL_dG = r1.w * dL_dalpha;
                                const float gdx = Gs * dx, gdy = Gs * dy;
                                const float dG_ddelx = -gdx * r1.x - gdy * r1.y;
                                const float dG_ddely = -gdy * r1.z - gdx * r1.y;
                                v[0] = dL_dG * dG_ddelx * ddelx_dx;
                                v[1] = dL_dG * dG_ddely * ddely_dy;
                                v[2] = -0.5f * gdx * dx * dL_dG;
                                v[3] = -0.5f * gdx * dy * dL_dG;
                                v[4] = -0.5f * gdy * dy * dL_dG;
                                v[5] = Gs * dL_dalpha;
                                v[6] = wgt * p.dLd;
                            }
                            const uint32_t pm = __ballot_sync(0xffffffffu, contrib);
                            if (pm) {
                                if (kTimingB) nA_pm++;
                                if (CH > 0) {
                                    ws->w[k][lane] = wgt;
                                    if (lane == 0) ws->pm[k] = pm;
                                    km |= 1u << k;
                                }
                                if (EMIT) {  // one 128-byte row of weights + {id, mask} per blended (block, instance)
                                    const size_t e = ebase[bi] + ecount[bi];
                                    args.list_w[e * 32 + lane] = wgt;
                                    if (lane == 0) args.list_meta[e] = make_uint2(st.gid[k], pm);
                                    ecount[bi]++;
                                }
                                if (do_geom) {
#pragma unroll
                                    for (int i = 0; i < kRedVals; i++) red[i * kRedSlots + nslots][lane] = v[i];
                                    if (lane == 0) red_gid[nslots] = st.gid[k];
                                    nslots++;
                                    if (nslots == kRedSlots) flush();
                                }
                            }
                        }
                    }
                }
                if (CH > 0) {
                    __syncwarp();
                    if (lane == 0) {
                        ws->km = km;
                        ws->last = last;
                        ws->first = first;
                        ws->work = work;
                        mbar_arrive(&ring.wfull[b][j]);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&ring.empty[s]);
            if (EMIT && last && lane == 0) {
#pragma unroll
                for (int bi = 0; bi < BPA; bi++) args.list_cnt[(size_t)etile * kBlocksPerTile + BPA * a + bi] = ecount[bi];
            }
            if (last && nslots > 0) flush();
            if (++s == kStages) { s = 0; parity ^= 1; }
            if (CH > 0 && ++j == kWSlots) { j = 0; wparity ^= 1; }
        }
        if (kTimingB && args.dbg && lane == 0) {
            long long* d = args.dbg + (blockIdx.x * 32 + warp) * 8;
            d[0] = clock64() - tA_total; d[1] = tA_full; d[2] = tA_wempty; d[3] = tA_flush; d[4] = nA_hits; d[5] = nA_pm;
        }
        if (CH > 0) {
#pragma unroll
            for (int bi = 0; bi < BPA; bi++) {
                const int b = BPA * a + bi;
                mbar_wait(&ring.wempty[b][j], wparity);
                if (lane == 0) {
                    ring.ws[b][j].work = -1;
                    ring.ws[b][j].km = 0;
                    mbar_arrive(&ring.wfull[b][j]);
                }
            }
        }
        return;
    }

    // ======================================================================== feature warps
    if (CH == 0) return;
    reg_inc<L::kRegsFeature>();
    {
        constexpr int LPR = CH > 0 ? CH / 4 : 32;
        constexpr int G = 32 / LPR;
        constexpr int NQ = 8 / G;
        const int b = warp - L::kFeatWarp0;
        const int grp = lane / LPR, cl = lane % LPR;
        // upstream feature gradient: [quad][pixel in quad][channel]; with F3DGS_FFMA2 the two pixels of a quad row share a
        // 64-bit register pair (they arrive adjacent from the 128-bit loads, as do their weights from the LDS.128), so one
        // paired FMA (weight pair x dO pair + g pair, fma2_rn) covers both; g.x / g.y collect the even / odd pixel columns
#if F3DGS_FFMA2
        float2 dO2[NQ][2][4];
#define DO(q, i, c) (((i) & 1) ? dO2[q][(i) >> 1][c].y : dO2[q][(i) >> 1][c].x)
#else
        float dO[NQ][4][4];
#define DO(q, i, c) dO[q][i][c]
#endif
        int s = 0, j = 0, ch0 = 0;
        uint32_t parity = 0, wparity = 0;
        long long tF_wfull = 0, tF_full = 0, tF_load = 0, tF_loop = 0, nF_k = 0;
        const long long tF_total = BTICK();
        for (;;) {
            { const long long t_ = BTICK(); mbar_wait(&ring.wfull[b][j], wparity); tF_wfull += BTICK() - t_; }
            const WSlot& ws = ring.ws[b][j];
            const int work = ws.work;
            if (work < 0) break;
            uint32_t km = ws.km;
            const long long tL_ = BTICK();
            if (ws.first) {
                const int tile = work / args.pa.chunks, chunk = work - tile * args.pa.chunks;
                const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
                const int bx0 = tile_x * 16 + (b & 1) * 8, by0 = tile_y * 16 + (b >> 1) * 4;
                ch0 = chunk * CH + cl * 4;
#pragma unroll
                for (int q = 0; q < NQ; q++)
#pragma unroll
                    for (int i = 0; i < 4; i++)
#pragma unroll
                        for (int c = 0; c < 4; c++) DO(q, i, c) = 0.f;
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const int ch = ch0 + c;
                    if (ch >= C) continue;
                    const float* plane = args.dL_dfeat_pix + (size_t)ch * HW;
                    if (G == 1 && (args.vec_io & 1)) {
#pragma unroll
                        for (int y = 0; y < 4; y++) {
                            const int yy = by0 + y;
                            if (yy >= H) continue;
#pragma unroll
                            for (int half = 0; half < 2; half++) {
                                const int xx = bx0 + half * 4;
                                if (xx >= W) continue;
                                const int qa = (y >> 1) * 4 + half * 2, i0 = (y & 1) * 2;
                                const float4 v = ld_nc_f4(plane + (size_t)yy * W + xx);
                                DO(qa % NQ, i0, c) = v.x;
                                DO(qa % NQ, i0 + 1, c) = v.y;
                                DO((qa + 1) % NQ, i0, c) = v.z;
                                DO((qa + 1) % NQ, i0 + 1, c) = v.w;
                            }
                        }
                    } else {
#pragma unroll
                        for (int qi = 0; qi < NQ; qi++) {
                            const int q = qi * G + grp;
#pragma unroll
                            for (int i = 0; i < 4; i++) {
                                const int xx = bx0 + (q & 3) * 2 + (i & 1), yy = by0 + (q >> 2) * 2 + (i >> 1);
                                if (xx < W && yy < H) DO(qi, i, c) = __ldg(plane + (size_t)yy * W + xx);
                            }
                        }
                    }
                }
            }
            tF_load += BTICK() - tL_;
            { const long long t_ = BTICK(); mbar_wait(&ring.full[s], parity); tF_full += BTICK() - t_; }
            if (kTimingB) nF_k += __popc(km);
            if (F3DGS_DIAG_NO_FMA) km = 0;
            const Stage<0>& st = ring.stage[s];
            const long long tK_ = BTICK();
            while (km) {
                const int k = __ffs(km) - 1;
                km &= km - 1;
                const uint32_t pm = ws.pm[k];
                const uint32_t gid = st.gid[k];
                float4 w4[NQ];
                if (L::kPrefetchW) {
#pragma unroll
                    for (int qi = 0; qi < NQ; qi++)
                        w4[qi] = *reinterpret_cast<const float4*>(&ws.w[k][4 * (qi * G + grp)]);
                }
#if F3DGS_FFMA2
                float2 gp[4];  // per channel: (sum over even pixel columns, sum over odd pixel columns)
#pragma unroll
                for (int c = 0; c < 4; c++) gp[c] = make_float2(0.f, 0.f);
#pragma unroll
                for (int qi = 0; qi < NQ; qi++) {
                    const int q = qi * G + grp;
                    if ((pm >> (4 * q)) & 0xFu) {
                        if (!L::kPrefetchW) w4[qi] = *reinterpret_cast<const float4*>(&ws.w[k][4 * q]);
                        const float2 w01 = make_float2(w4[qi].x, w4[qi].y), w23 = make_float2(w4[qi].z, w4[qi].w);
#if F3DGS_PAIR_SKIP
                        if ((pm >> (4 * q)) & 0x3u)
#endif
                        {
#pragma unroll
                            for (int c = 0; c < 4; c++) gp[c] = fma2_rn(w01, dO2[qi][0][c], gp[c]);
                        }
#if F3DGS_PAIR_SKIP
                        if ((pm >> (4 * q)) & 0xCu)
#endif
                        {
#pragma unroll
                            for (int c = 0; c < 4; c++) gp[c] = fma2_rn(w23, dO2[qi][1][c], gp[c]);
                        }
                    }
                }
                float g0 = gp[0].x + gp[0].y, g1 = gp[1].x + gp[1].y, g2 = gp[2].x + gp[2].y, g3 = gp[3].x + gp[3].y;
#else
                float g0 = 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f;
#pragma unroll
                for (int qi = 0; qi < NQ; qi++) {
                    const int q = qi * G + grp;
                    if ((pm >> (4 * q)) & 0xFu) {
                        if (!L::kPrefetchW) w4[qi] = *reinterpret_cast<const float4*>(&ws.w[k][4 * q]);
                        const float wv[4] = {w4[qi].x, w4[qi].y, w4[qi].z, w4[qi].w};
#pragma unroll
                        for (int i = 0; i < 4; i++) {
                            g0 = fmaf(wv[i], dO[qi][i][0], g0);
                            g1 = fmaf(wv[i], dO[qi][i][1], g1);
                            g2 = fmaf(wv[i], dO[qi][i][2], g2);
                            g3 = fmaf(wv[i], dO[qi][i][3], g3);
                        }
                    }
                }
#endif
#pragma unroll
                for (int o = LPR; o < 32; o <<= 1) {
                    g0 += __shfl_xor_sync(0xffffffffu, g0, o);
                    g1 += __shfl_xor_sync(0xffffffffu, g1, o);
                    g2 += __shfl_xor_sync(0xffffffffu, g2, o);
                    g3 += __shfl_xor_sync(0xffffffffu, g3, o);
                }
                if (grp == 0 && ch0 < C) {
                    float* dst = args.dL_dfeature + (size_t)gid * C + ch0;
                    if (F3DGS_DIAG_NO_FEAT_RED) {
                        if (g0 + g1 + g2 + g3 == 123456.789f) red_add_f1(dst, g0);  // keeps the FMAs alive
                    } else if (args.vec_io & 2) {
                        red_add_f4(dst, make_float4(g0, g1, g2, g3));
                    } else {
                        red_add_f1(dst, g0);
                        if (ch0 + 1 < C) red_add_f1(dst + 1, g1);
                        if (ch0 + 2 < C) red_add_f1(dst + 2, g2);
                        if (ch0 + 3 < C) red_add_f1(dst + 3, g3);
                    }
                }
            }
            __syncwarp();
            tF_loop += BTICK() - tK_;
            if (lane == 0) {
                mbar_arrive(&ring.wempty[b][j]);
                mbar_arrive(&ring.empty[s]);
            }
            if (++s == kStages) { s = 0; parity ^= 1; }
            if (++j == kWSlots) { j = 0; wparity ^= 1; }
        }
        if (kTimingB && args.dbg && lane == 0) {
            long long* d = args.dbg + (blockIdx.x * 32 + warp) * 8;
            d[0] = clock64() - tF_total; d[1] = tF_wfull; d[2] = tF_full; d[3] = tF_load; d[4] = nF_k; d[5] = tF_loop;
        }
    }
}


template <int CH, int BPA>
static cudaError_t launch_bwd_t(const ViewParams& vp, BwdArgs a, cudaStream_t s) {
    const size_t smem = sizeof(BwdSmem);
    // the opt-in to > 48 KB of dynamic shared memory is per device (context): remember it per device ordinal, so that one
    // process driving several GPUs works too
    static std::atomic<int> sms_of_device[64];  // zero-initialised; set once per device (idempotent)
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    if (sms_of_device[dev].load() == 0) {
        cudaError_t e = cudaFuncSetAttribute(composite_bwd_kernel<CH, BPA>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem);
        if (e != cudaSuccess) return e;
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sms_of_device[dev].store(n > 0 ? n : 132);
    }
    const int num_sms = sms_of_device[dev].load();
    a.pa.chunks = CH > 0 ? (vp.C + CH - 1) / CH : 1;
    a.vec_io = 0;
    if (vp.W % 4 == 0 && (reinterpret_cast<uintptr_t>(a.dL_dfeat_pix) & 15) == 0) a.vec_io |= 1;
    if (vp.C % 4 == 0 && (reinterpret_cast<uintptr_t>(a.dL_dfeature) & 15) == 0) a.vec_io |= 2;
    cudaError_t e = cudaMemsetAsync(a.pa.work_counter, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    const int grid = min(a.pa.num_tiles * a.pa.chunks, num_sms);
    static long long* dbg = nullptr;
    const bool timing = kTimingB && getenv("F3DGS_TIMING") != nullptr;  // debug aid: per-role cycle breakdown on stderr
    if (timing && !dbg) cudaMalloc(&dbg, 256 * 32 * 8 * sizeof(long long));
    a.dbg = timing ? dbg : nullptr;
    if (timing) cudaMemsetAsync(dbg, 0, 256 * 32 * 8 * sizeof(long long), s);
    composite_bwd_kernel<CH, BPA><<<grid, Layout<BPA>::kThreads, smem, s>>>(a);
    g_launches++;
    if (timing) {
        static long long host[256 * 32 * 8];
        cudaMemcpyAsync(host, dbg, sizeof(host), cudaMemcpyDeviceToHost, s);
        cudaStreamSynchronize(s);
        const int nA = Layout<BPA>::kAlphaWarps, f0 = Layout<BPA>::kFeatWarp0;
        double A[6] = {0, 0, 0, 0, 0, 0}, F[6] = {0, 0, 0, 0, 0, 0};
        for (int c = 0; c < grid; c++) {
            for (int w = 0; w < nA; w++) for (int i = 0; i < 6; i++) A[i] += host[(c * 32 + kAlphaWarp0 + w) * 8 + i];
            for (int w = 0; w < 8; w++) for (int i = 0; i < 6; i++) F[i] += host[(c * 32 + f0 + w) * 8 + i];
        }
        fprintf(stderr, "[f3dgs timing bwd CH=%d BPA=%d] per-warp mean cycles: alpha total %.0f wait_full %.0f wait_wempty %.0f flush %.0f hits %.0f pm %.0f | feature total %.0f wait_wfull %.0f wait_full %.0f tile_load %.0f k %.0f k_loop %.0f\n",
                CH, BPA, A[0] / (grid * nA), A[1] / (grid * nA), A[2] / (grid * nA), A[3] / (grid * nA), A[4] / (grid * nA),
                A[5] / (grid * nA), F[0] / (grid * 8), F[1] / (grid * 8), F[2] / (grid * 8), F[3] / (grid * 8), F[4] / (grid * 8), F[5] / (grid * 8));
    }
    return cudaGetLastError();
}

// Geometric-gradient pass of the two-pass mode with the slim layout (F3DGS_SPLIT=2): C = 0 kernel, two CTAs per SM.
cudaError_t launch_composite_bwd_geom_slim(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                           const SplatRec* rec, const float* bg, const float* final_T,
                                           const uint32_t* n_contrib, const float* dL_dpix, const float* dL_ddepth,
                                           float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                                           float* dL_dz, int* work_counter, cudaStream_t s, float* list_w,
                                           uint2* list_meta, uint32_t* list_cnt) {
    using SMEM = BwdSmemT<RingSlim>;
    const bool emit = list_w != nullptr;
    const size_t smem = sizeof(SMEM);
    static std::atomic<int> sms_of_device[64];  // zero-initialised; set once per device (idempotent)
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    if (sms_of_device[dev].load() == 0) {
        cudaError_t e = cudaFuncSetAttribute(composite_bwd_kernel<0, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(composite_bwd_kernel<0, 1, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem);
        if (e != cudaSuccess) return e;
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sms_of_device[dev].store(n > 0 ? n : 132);
    }
    BwdArgs a;
    a.pa.ranges = ranges; a.pa.point_list = point_list; a.pa.rec = rec; a.pa.features = nullptr;
    a.pa.n_contrib = n_contrib; a.pa.work_counter = work_counter;
    a.pa.W = vp.W; a.pa.H = vp.H; a.pa.C = 0;
    a.pa.tiles_x = (int)vp.grid_x; a.pa.num_tiles = (int)(vp.grid_x * vp.grid_y); a.pa.chunks = 1; a.pa.use_bulk = 0;
    a.bg = bg; a.final_T = final_T; a.n_contrib = n_contrib; a.dL_dpix = dL_dpix; a.dL_dfeat_pix = nullptr;
    a.dL_ddepth = dL_ddepth; a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic; a.dL_dopacity = dL_dopacity;
    a.dL_dcolor = dL_dcolor; a.dL_dfeature = nullptr; a.dL_dz = dL_dz; a.vec_io = 0; a.dbg = nullptr;
    a.list_w = list_w; a.list_meta = list_meta; a.list_cnt = list_cnt;
    cudaError_t e = cudaMemsetAsync(work_counter, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    const int grid = min(a.pa.num_tiles, kSlimCtas * sms_of_device[dev].load());
    if (emit)
        composite_bwd_kernel<0, 1, true, true><<<grid, (kAlphaWarp0 + Layout<1>::kAlphaWarps) * 32, smem, s>>>(a);
    else
        composite_bwd_kernel<0, 1, true><<<grid, (kAlphaWarp0 + Layout<1>::kAlphaWarps) * 32, smem, s>>>(a);
    g_launches++;
    return cudaGetLastError();
}

#define F3DGS_BWD_DISPATCH(CHV) launch_bwd_t<CHV, 1>(vp, a, s)

cudaError_t launch_composite_bwd(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                 const SplatRec* rec, const float* bg, const float* final_T,
                                 const uint32_t* n_contrib, const float* dL_dpix, const float* dL_dfeat_pix,
                                 const float* dL_ddepth, float* dL_dmean2D, float* dL_dconic,
                                 float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dz,
                                 int* work_counter, cudaStream_t s) {
    BwdArgs a;
    a.pa.ranges = ranges; a.pa.point_list = point_list; a.pa.rec = rec; a.pa.features = nullptr;
    a.pa.n_contrib = n_contrib; a.pa.work_counter = work_counter;
    a.pa.W = vp.W; a.pa.H = vp.H; a.pa.C = vp.C;
    a.pa.tiles_x = (int)vp.grid_x; a.pa.num_tiles = (int)(vp.grid_x * vp.grid_y); a.pa.chunks = 1;
    a.pa.use_bulk = 0;
    a.bg = bg; a.final_T = final_T; a.n_contrib = n_contrib; a.dL_dpix = dL_dpix; a.dL_dfeat_pix = dL_dfeat_pix;
    a.dL_ddepth = dL_ddepth; a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic; a.dL_dopacity = dL_dopacity;
    a.dL_dcolor = dL_dcolor; a.dL_dfeature = dL_dfeature; a.dL_dz = dL_dz; a.vec_io = 0; a.dbg = nullptr;
    a.list_w = nullptr; a.list_meta = nullptr; a.list_cnt = nullptr;
    if (vp.C == 0) return F3DGS_BWD_DISPATCH(0);
    if (vp.C <= 32) return F3DGS_BWD_DISPATCH(32);
    if (vp.C <= 64) return F3DGS_BWD_DISPATCH(64);
    return F3DGS_BWD_DISPATCH(128);
}

}  // namespace f3dgs
