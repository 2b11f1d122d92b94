// Forward tile composite: front-to-back alpha blend of RGB, depth and a C-wide feature vector.
// Reference: forward.cu:261-396 (renderCUDA<3>), semantics restated in SURVEY.md A.4.
//
// Per pixel the arithmetic that decides WHAT is blended (power, alpha, T, the 1/255 and 1e-4
// tests, n_contrib, final_T) and the RGB/depth accumulation are the reference's expressions
// compiled by the same compiler (see common.cuh), so those outputs are bit-identical.  The feature
// accumulation uses acc = fma(f, alpha*T, acc) instead of fma(T, alpha*f, acc): one rounding
// differs per term (<= 1 ulp of the term), which halves the FMA-pipe work of the hot loop.
//
// Roles (composite_common.cuh): producer -> alpha warps -> feature warps, persistent over tiles.
//   alpha warp b   lane = pixel of block b.  For every staged instance whose footprint reaches
//                  the block: alpha, T update, RGB/depth accumulate; publishes w = alpha*T as a
//                  [instance][pixel] tile + a 32-bit "which pixels blended" mask per instance.
//   feature warp b lane = float4 of channels.  acc[pixel][4] += w[pixel] * f[4] for the pixels in
//                  the mask, 2x2-pixel quads at a time: one broadcast LDS.128 of weights feeds
//                  16 FFMAs; the feature float4 is loaded once per instance.  All 32 pixels x 4
//                  channels (= 128 accumulators per lane at CH = 128) live in registers.
//   TC feature warps (launch_composite_fwd_tc): the same roles, with the block's contraction
//                  D[ch, px] = sum_k f[k, ch] * w[k, px] on the tensor cores: per 8 staged instances
//                  three mma.sync m16n8k8 TF32 products per 16 channels x 8 pixels (3xTF32, tc_common.cuh),
//                  fp32 accumulators in registers (CH x 32 per warp, as in the fp32 loop).
// Channel counts above 128 are split into chunks of 128 (extra work items); chunk 0 also writes
// colour, depth, final_T and n_contrib.
#include <cstdio>
#include <cstdlib>

#include "composite_common.cuh"
#include "tc_common.cuh"

namespace f3dgs {

#ifndef F3DGS_TIMING_BUILD
#define F3DGS_TIMING_BUILD 0   // build.py sets 1 when env F3DGS_TIMING_BUILD=1: per-role cycle counters (see tools/stage_times.py)
#endif
#ifndef F3DGS_FWD_COPYWARP
#define F3DGS_FWD_COPYWARP 1
#endif
#ifndef F3DGS_FWD_A1
#define F3DGS_FWD_A1 64
#define F3DGS_FWD_F1 152
#endif
#ifndef F3DGS_FFMA2
#define F3DGS_FFMA2 1          // 1: feature loop on paired accumulators (fma2_rn, common.cuh: two scalar fma.rn on sm_90)
#endif
#ifndef F3DGS_DIAG_NO_FMA
#define F3DGS_DIAG_NO_FMA 0    // diagnostic builds only (WRONG RESULTS): feature warps consume their slots without the FMAs
#endif
#ifndef F3DGS_PAIR_SKIP
#define F3DGS_PAIR_SKIP 1      // 1 (with F3DGS_FFMA2): skip the paired FMAs of a quad row whose two pixels did not blend
#endif
#ifndef F3DGS_FEAT_PREFETCH
#define F3DGS_FEAT_PREFETCH 1  // 1: software-pipeline the sparse feature loop by one instance (mask + feature float4)
#endif
static constexpr bool kTiming = F3DGS_TIMING_BUILD != 0;
#define TICK() ((kTiming && args.dbg) ? clock64() : 0ll)

struct FwdArgs {
    ProducerArgs pa;
    const float* bg;
    float* final_T;
    uint32_t* n_contrib;
    float* out_color;
    float* out_feature;
    float* out_depth;
    int vec_store;
    long long* dbg;  // F3DGS_TIMING=1: per-warp cycle counters [cta][warp][8], else nullptr
};

// Forward register budget.  BPA == 1 (20 warps, launched at 96 regs/thread = 61440 in the CTA pool):
// 4x32x40 + 8x32x64 + 8x32x152 = 60416, feature warps run the sparse quad loop.  The alternative 40/48/168 with the
// dense hoisted loop (-DF3DGS_FWD_A1=48 -DF3DGS_FWD_F1=168) is kept as a build option; its extra FMA issue competes
// with the alpha warps sharing the SMSP.
// The TC feature warps hold the same CH x 32 accumulators plus the split operand fragments of one K = 8 step:
// 4x32x40 + 8x32x56 + 8x32x160 = 60416.
template <int BPA, bool TC = false>
struct FwdLayout : Layout<BPA> {
    static constexpr int kRegsAlpha = TC ? 56 : (BPA == 2 ? 104 : F3DGS_FWD_A1);
    static constexpr int kRegsFeature = TC ? 160 : (BPA == 2 ? 184 : F3DGS_FWD_F1);
    static constexpr bool kPrefetchW = BPA == 2 || F3DGS_FWD_F1 >= 168;
};

template <int CH, int BPA, bool TC>
__global__ void __launch_bounds__(Layout<BPA>::kThreads, 1)
composite_fwd_kernel(const FwdArgs args) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using RING = RingV2<CH>;
    RING& ring = *reinterpret_cast<RING*>(smem_raw);
    // The warp index goes through a shuffle so that ptxas knows it is warp-uniform: role branches, ring/slot addresses
    // and everything loaded from them (instance masks, work ids) then live in uniform registers, the per-quad branches
    // of the feature loop need no BSSY/BSYNC reconvergence pair, and nothing is re-derived from SR_TID inside the loops.
    const int warp = F3DGS_UNIFORM_WARP ? __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0) : (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int W = args.pa.W, H = args.pa.H, C = args.pa.C;
    const size_t HW = (size_t)H * W;

    using L = FwdLayout<BPA, TC>;
    constexpr bool kCopyWarp = CH > 0 && F3DGS_FWD_COPYWARP;  // see producer_loop<>
    ring_init<CH>(ring, CH > 0 ? L::kAlphaWarps + kBlocksPerTile : L::kAlphaWarps, CH > 0, kCopyWarp ? 2 : 1);
    __syncthreads();

    // ======================================================================== producer group
    if (warp < kAlphaWarp0) {
        reg_dec<L::kRegsProducer>();
        if (warp == kProducerWarp) {
            const long long t0 = TICK();
            producer_loop<CH, false, kCopyWarp, RING>(ring, args.pa);
            if (kTiming && args.dbg && (threadIdx.x & 31) == 0) args.dbg[(blockIdx.x * 32 + warp) * 8 + 0] = clock64() - t0;
        } else if (kCopyWarp && warp == kProducerWarp + 1) {
            if constexpr (kCopyWarp) copy_loop<CH>(ring, args.pa);
        }
        return;
    }

    // ======================================================================== alpha warps
    if (warp < L::kFeatWarp0) {
        reg_dec<L::kRegsAlpha>();
        const int a = warp - kAlphaWarp0;  // owns blocks BPA*a .. BPA*a + BPA-1
        int s = 0, j = 0;
        uint32_t parity = 0, wparity = 1;  // wempty: fresh barrier falls through on parity 1
        float T[BPA], Cr[BPA], Cg[BPA], Cb[BPA], Dp[BPA], pxf[BPA], pyf[BPA], fbx0[BPA], fby0[BPA];
        uint32_t last_contrib[BPA];
        int px[BPA], py[BPA], chunk = 0;
        bool done[BPA], inside[BPA], blk_done[BPA];
#pragma unroll
        for (int bi = 0; bi < BPA; bi++) {
            T[bi] = 1.f; Cr[bi] = Cg[bi] = Cb[bi] = Dp[bi] = 0.f; pxf[bi] = pyf[bi] = fbx0[bi] = fby0[bi] = 0.f;
            last_contrib[bi] = 0; px[bi] = py[bi] = 0; done[bi] = true; inside[bi] = false; blk_done[bi] = true;
        }
        long long tA_full = 0, tA_wempty = 0, tA_total = TICK(), nA_stage = 0, nA_hits = 0;
        for (;;) {
            { const long long t_ = TICK(); mbar_wait(&ring.full[s], parity); tA_full += TICK() - t_; }
            nA_stage++;
            Stage<CH>& st = ring.stage[s];
            const uint32_t n = st.n, last = st.last, first = st.first;
            const int work = st.work;
            if (work < 0) break;
            if (first) {
                const int tile = work / args.pa.chunks;
                chunk = work - tile * args.pa.chunks;
                const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
#pragma unroll
                for (int bi = 0; bi < BPA; bi++) {
                    const int b = BPA * a + bi;
                    const int bx0 = tile_x * 16 + (b & 1) * 8, by0 = tile_y * 16 + (b >> 1) * 4;
                    px[bi] = bx0 + lane_px(lane);
                    py[bi] = by0 + lane_py(lane);
                    inside[bi] = px[bi] < W && py[bi] < H;
                    pxf[bi] = (float)px[bi]; pyf[bi] = (float)py[bi];
                    fbx0[bi] = (float)bx0; fby0[bi] = (float)by0;
                    T[bi] = 1.f; Cr[bi] = Cg[bi] = Cb[bi] = Dp[bi] = 0.f;
                    last_contrib[bi] = 0;
                    done[bi] = !inside[bi];
                    blk_done[bi] = __all_sync(0xffffffffu, done[bi]);
                    if (blk_done[bi] && lane == 0) atomicOr(&ring.done_mask[st.done_slot], 1u << b);
                }
            }
            if constexpr (BPA == 2) {
                // Two blocks per alpha warp, advanced in lock-step.  One trip takes up to two hits of each block:
                // all operand loads first, then the four alpha evaluations written "transposed" (one operation
                // across the four instances at a time) so their LDS -> FFMA -> MUFU.EX2 chains overlap, then the
                // two blocks' T recurrences as two independent dependency chains.
                WSlot* wsl[2] = {&ring.ws[2 * a][j], &ring.ws[2 * a + 1][j]};
                if (CH > 0) {
                    const long long t_ = TICK();
                    mbar_wait(&ring.wempty[2 * a][j], wparity);
                    mbar_wait(&ring.wempty[2 * a + 1][j], wparity);
                    tA_wempty += TICK() - t_;
                }
                uint32_t kmv[2] = {0u, 0u};
                if (n > 0 && !(blk_done[0] && blk_done[1])) {
                    bool h0 = false, h1 = false;
                    if (lane < n) {
                        const float4 r0 = st.rec0[lane];
                        const bool hy = (r0.y + r0.w >= fby0[0]) && (r0.y - r0.w <= fby0[0] + 3.f);  // same pixel rows
                        h0 = hy && (r0.x + r0.z >= fbx0[0]) && (r0.x - r0.z <= fbx0[0] + 7.f);
                        h1 = hy && (r0.x + r0.z >= fbx0[1]) && (r0.x - r0.z <= fbx0[1] + 7.f);
                    }
                    uint32_t amv[2];
                    amv[0] = blk_done[0] ? 0u : __ballot_sync(0xffffffffu, h0);
                    amv[1] = blk_done[1] ? 0u : __ballot_sync(0xffffffffu, h1);
                    nA_hits += __popc(amv[0]) + __popc(amv[1]);
                    while (amv[0] | amv[1]) {
                        int kk[4];   // e = 2*u + bi
                        bool vk[4];
#pragma unroll
                        for (int u = 0; u < 2; u++)
#pragma unroll
                            for (int bi = 0; bi < 2; bi++) {
                                const int e = 2 * u + bi;
                                vk[e] = amv[bi] != 0;
                                kk[e] = vk[e] ? (__ffs(amv[bi]) - 1) : 0;
                                amv[bi] &= amv[bi] - 1;
                            }
                        float2 xy[4];
                        float4 co[4], r2[4];
                        uint32_t lp[4];
#pragma unroll
                        for (int e = 0; e < 4; e++) {
                            xy[e] = *reinterpret_cast<const float2*>(&st.rec0[kk[e]]);
                            co[e] = st.rec1[kk[e]];
                            r2[e] = st.rec2[kk[e]];
                            lp[e] = st.listpos[kk[e]];
                        }
                        asm volatile("" ::: "memory");
                        float dx[4], dy[4], pw[4], av[4], al[4];
#pragma unroll
                        for (int e = 0; e < 4; e++) { dx[e] = xy[e].x - pxf[e & 1]; dy[e] = xy[e].y - pyf[e & 1]; }
                        // same expression trees as reference forward.cu:340-351 (see common.cuh)
#pragma unroll
                        for (int e = 0; e < 4; e++)
                            pw[e] = -0.5f * (co[e].x * dx[e] * dx[e] + co[e].z * dy[e] * dy[e]) - co[e].y * dx[e] * dy[e];
#pragma unroll
                        for (int e = 0; e < 4; e++) av[e] = fminf(0.99f, co[e].w * expf(pw[e]));
#pragma unroll
                        for (int e = 0; e < 4; e++)
                            al[e] = (vk[e] && !(pw[e] > 0.0f) && !(av[e] < 1.0f / 255.0f)) ? av[e] : 0.f;
#pragma unroll
                        for (int u = 0; u < 2; u++) {
                            float wgt[2];
                            bool blend[2];
#pragma unroll
                            for (int bi = 0; bi < 2; bi++) {
                                const int e = 2 * u + bi;
                                const float alpha = al[e];
                                const float test_T = T[bi] * (1 - alpha);
                                const bool act = !done[bi] && alpha > 0.f;
                                const bool stop = act && (test_T < 0.0001f);  // reference: done = true, not blended
                                blend[bi] = act && !stop;
                                done[bi] = done[bi] || stop;
                                wgt[bi] = blend[bi] ? alpha * T[bi] : 0.f;
                                const float nCr = Cr[bi] + r2[e].x * alpha * T[bi];  // reference forward.cu:362-368
                                const float nCg = Cg[bi] + r2[e].y * alpha * T[bi];
                                const float nCb = Cb[bi] + r2[e].z * alpha * T[bi];
                                const float nDp = Dp[bi] + r2[e].w * (alpha * T[bi]);
                                Cr[bi] = blend[bi] ? nCr : Cr[bi];
                                Cg[bi] = blend[bi] ? nCg : Cg[bi];
                                Cb[bi] = blend[bi] ? nCb : Cb[bi];
                                Dp[bi] = blend[bi] ? nDp : Dp[bi];
                                T[bi] = blend[bi] ? test_T : T[bi];
                                last_contrib[bi] = blend[bi] ? lp[e] : last_contrib[bi];
                            }
#pragma unroll
                            for (int bi = 0; bi < 2; bi++) {
                                const int e = 2 * u + bi;
                                const uint32_t pm = __ballot_sync(0xffffffffu, blend[bi]);
                                if (CH > 0 && vk[e]) {  // warp-uniform
                                    wsl[bi]->w[kk[e]][lane] = wgt[bi];
                                    if (lane == 0) wsl[bi]->pm[kk[e]] = pm;
                                    kmv[bi] |= (pm ? 1u : 0u) << kk[e];
                                }
                            }
                        }
                    }
#pragma unroll
                    for (int bi = 0; bi < 2; bi++)
                        if (!blk_done[bi] && __all_sync(0xffffffffu, done[bi])) {
                            blk_done[bi] = true;
                            if (lane == 0) atomicOr(&ring.done_mask[st.done_slot], 1u << (2 * a + bi));
                        }
                }
                if (CH > 0) {
                    __syncwarp();
                    if (lane == 0) {
#pragma unroll
                        for (int bi = 0; bi < 2; bi++) {
                            wsl[bi]->km = kmv[bi]; wsl[bi]->last = last; wsl[bi]->first = first; wsl[bi]->work = work;
                            mbar_arrive(&ring.wfull[2 * a + bi][j]);
                        }
                    }
                }
            } else {
#pragma unroll
            for (int bi = 0; bi < BPA; bi++) {
                const int b = BPA * a + bi;
                WSlot* ws = &ring.ws[b][j];
                if (CH > 0) { const long long t_ = TICK(); mbar_wait(&ring.wempty[b][j], wparity); tA_wempty += TICK() - t_; }
                uint32_t km = 0;
                if (!blk_done[bi] && n > 0) {
                    bool hit = false;
                    if (lane < n) {
#if F3DGS_EXACT_CULL
                        hit = footprint_hits_rect(st.rec0[lane], st.rec1[lane], fbx0[bi], fbx0[bi] + 7.f, fby0[bi],
                                                  fby0[bi] + 3.f);
#else
                        const float4 r0 = st.rec0[lane];
                        hit = (r0.x + r0.z >= fbx0[bi]) && (r0.x - r0.z <= fbx0[bi] + 7.f) &&
                              (r0.y + r0.w >= fby0[bi]) && (r0.y - r0.w <= fby0[bi] + 3.f);
#endif
                    }
                    uint32_t am = __ballot_sync(0xffffffffu, hit);
                    nA_hits += __popc(am);
                    while (am) {
                        // Up to 4 instances per trip.  Everything is branch-free so that the four alpha
                        // evaluations (LDS -> power -> expf) interleave in the pipeline; only the short
                        // T / done recurrence is serial.
                        int kk[4];
                        bool vk[4];
                        float al[4];
#pragma unroll
                        for (int u = 0; u < 4; u++) {
                            vk[u] = am != 0;
                            kk[u] = vk[u] ? (__ffs(am) - 1) : 0;
                            am &= am - 1;
                        }
#pragma unroll
                        for (int u = 0; u < 4; u++) {
                            const float4 r0 = st.rec0[kk[u]];
                            const float4 r1 = st.rec1[kk[u]];
                            // same expression trees as reference forward.cu:340-351 (see common.cuh)
                            const float dx = r0.x - pxf[bi], dy = r0.y - pyf[bi];
                            const float power = -0.5f * (r1.x * dx * dx + r1.z * dy * dy) - r1.y * dx * dy;
                            const float av = fminf(0.99f, r1.w * expf(power));
                            al[u] = (vk[u] && !(power > 0.0f) && !(av < 1.0f / 255.0f)) ? av : 0.f;
                        }
#pragma unroll
                        for (int u = 0; u < 4; u++) {
                            if (!vk[u]) break;  // warp-uniform, only in the last trip
                            const float4 r2 = st.rec2[kk[u]];
                            const uint32_t lp = st.listpos[kk[u]];
                            const float alpha = al[u];
                            const float test_T = T[bi] * (1 - alpha);
                            const bool act = !done[bi] && alpha > 0.f;
                            const bool stop = act && (test_T < 0.0001f);  // reference: done = true, not blended
                            const bool blend = act && !stop;
                            done[bi] = done[bi] || stop;
                            const float wgt = blend ? alpha * T[bi] : 0.f;
                            const float nCr = Cr[bi] + r2.x * alpha * T[bi];  // reference forward.cu:362-368
                            const float nCg = Cg[bi] + r2.y * alpha * T[bi];
                            const float nCb = Cb[bi] + r2.z * alpha * T[bi];
                            const float nDp = Dp[bi] + r2.w * (alpha * T[bi]);
                            Cr[bi] = blend ? nCr : Cr[bi];
                            Cg[bi] = blend ? nCg : Cg[bi];
                            Cb[bi] = blend ? nCb : Cb[bi];
                            Dp[bi] = blend ? nDp : Dp[bi];
                            T[bi] = blend ? test_T : T[bi];
                            last_contrib[bi] = blend ? lp : last_contrib[bi];
                            const uint32_t pm = __ballot_sync(0xffffffffu, blend);
                            if (CH > 0) {
                                ws->w[kk[u]][lane] = wgt;
                                if (lane == 0) ws->pm[kk[u]] = pm;
                                km |= (pm ? 1u : 0u) << kk[u];
                            }
                        }
                    }
                    if (__all_sync(0xffffffffu, done[bi])) {
                        blk_done[bi] = true;
                        if (lane == 0) atomicOr(&ring.done_mask[st.done_slot], 1u << b);
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
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&ring.empty[s]);
            if (last && chunk == 0) {
#pragma unroll
                for (int bi = 0; bi < BPA; bi++)
                    if (inside[bi]) {
                        const size_t pix = (size_t)py[bi] * W + px[bi];
                        args.final_T[pix] = T[bi];
                        args.n_contrib[pix] = last_contrib[bi];
                        args.out_color[pix] = Cr[bi] + T[bi] * args.bg[0];  // reference forward.cu:389
                        args.out_color[HW + pix] = Cg[bi] + T[bi] * args.bg[1];
                        args.out_color[2 * HW + pix] = Cb[bi] + T[bi] * args.bg[2];
                        args.out_depth[pix] = Dp[bi];
                    }
            }
            if (++s == kStages) { s = 0; parity ^= 1; }
            if (CH > 0 && ++j == kWSlots) { j = 0; wparity ^= 1; }
        }
        if (kTiming && args.dbg && lane == 0) {
            long long* d = args.dbg + (blockIdx.x * 32 + warp) * 8;
            d[0] = clock64() - tA_total; d[1] = tA_full; d[2] = tA_wempty; d[3] = nA_stage; d[4] = nA_hits;
        }
        if (CH > 0) {  // tell the feature warps of these blocks that the work is over
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
    if constexpr (TC) {
        // Tensor-core contraction.  B column n of n-tile ni is pixel (x = 2 ni + (n & 1), y = n >> 1) of the block, so the
        // accumulators of a lane (columns 2t, 2t + 1 of the four n-tiles) are the 8 pixels of block row t.  Instances of
        // the stage that did not blend in this block (km bit clear) and rows past the stage's end enter as zeros.
        constexpr int MT = CH / 16;  // m-tiles of 16 channels
        const int b = warp - L::kFeatWarp0;
        const int g = lane >> 2, t = lane & 3;
        int bcol[4];  // column of ws.w (alpha-warp lane, see lane_px / lane_py) holding pixel (2 ni + (g & 1), g >> 1)
#pragma unroll
        for (int ni = 0; ni < 4; ni++) bcol[ni] = ((g >> 2) << 4) | (ni << 2) | (((g >> 1) & 1) << 1) | (g & 1);
        float d[MT][4][4];
#pragma unroll
        for (int mi = 0; mi < MT; mi++)
#pragma unroll
            for (int ni = 0; ni < 4; ni++)
#pragma unroll
                for (int e = 0; e < 4; e++) d[mi][ni][e] = 0.f;
        int s = 0, j = 0;
        uint32_t parity = 0, wparity = 0;
        for (;;) {
            mbar_wait(&ring.wfull[b][j], wparity);
            const WSlot& ws = ring.ws[b][j];
            const int work = ws.work;
            if (work < 0) break;
            const uint32_t km = ws.km, last = ws.last;
            mbar_wait(&ring.full[s], parity);  // feature rows landed
            const Stage<CH>& st = ring.stage[s];
#pragma unroll 1
            for (int k0 = 0; k0 < kStageEntries; k0 += 8) {
                const uint32_t kb = (km >> k0) & 0xFFu;
                if (!kb) continue;  // warp-uniform
                const int ka = k0 + t, kc = ka + 4;
                const bool va = (kb >> t) & 1u, vc = (kb >> (t + 4)) & 1u;
                float bw[4][2];  // raw weights; the hi / lo split is redone at each use (registers go to the accumulators)
#pragma unroll
                for (int ni = 0; ni < 4; ni++) {
                    bw[ni][0] = va ? ws.w[ka][bcol[ni]] : 0.f;
                    bw[ni][1] = vc ? ws.w[kc][bcol[ni]] : 0.f;
                }
#pragma unroll
                for (int mi = 0; mi < MT; mi++) {
                    const int c0 = 16 * mi + g;
                    const float f[4] = {va ? st.feat[ka][c0] : 0.f, va ? st.feat[ka][c0 + 8] : 0.f,
                                        vc ? st.feat[kc][c0] : 0.f, vc ? st.feat[kc][c0 + 8] : 0.f};
                    uint32_t ah[4], al[4];
#pragma unroll
                    for (int r = 0; r < 4; r++) {
                        const float hi = tf32_hi(f[r]);
                        ah[r] = __float_as_uint(hi);
                        al[r] = __float_as_uint(f[r] - hi);
                    }
#pragma unroll
                    for (int ni = 0; ni < 4; ni++) {
                        uint32_t bh[2], bl[2];
#pragma unroll
                        for (int r = 0; r < 2; r++) {
                            const float hi = tf32_hi(bw[ni][r]);
                            bh[r] = __float_as_uint(hi);
                            bl[r] = __float_as_uint(bw[ni][r] - hi);
                        }
                        mma_tf32_16x8x8(d[mi][ni], ah, bh);
                        mma_tf32_16x8x8(d[mi][ni], ah, bl);
                        mma_tf32_16x8x8(d[mi][ni], al, bh);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&ring.wempty[b][j]);
                mbar_arrive(&ring.empty[s]);
            }
            if (last) {
                // ---- epilogue: lane (g, t) writes channels 16 mi + g (+ 8) of block row t, 8 pixels each
                const int tile = work / args.pa.chunks, chunk = work - tile * args.pa.chunks;
                const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
                const int bx0 = tile_x * 16 + (b & 1) * 8, yy = tile_y * 16 + (b >> 1) * 4 + t;
                if (yy < H) {
#pragma unroll
                    for (int mi = 0; mi < MT; mi++)
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const int ch = chunk * CH + 16 * mi + g + 8 * h;
                            float* row = args.out_feature + (size_t)ch * HW + (size_t)yy * W + bx0;
                            if (ch >= C) {
                            } else if ((args.vec_store & 1) && bx0 + 8 <= W) {
                                st_na_f4(row, make_float4(d[mi][0][2 * h], d[mi][0][2 * h + 1], d[mi][1][2 * h],
                                                          d[mi][1][2 * h + 1]));
                                st_na_f4(row + 4, make_float4(d[mi][2][2 * h], d[mi][2][2 * h + 1], d[mi][3][2 * h],
                                                              d[mi][3][2 * h + 1]));
                            } else {
#pragma unroll
                                for (int ni = 0; ni < 4; ni++)
#pragma unroll
                                    for (int e = 0; e < 2; e++)
                                        if (bx0 + 2 * ni + e < W) row[2 * ni + e] = d[mi][ni][2 * h + e];
                            }
                        }
                }
#pragma unroll
                for (int mi = 0; mi < MT; mi++)
#pragma unroll
                    for (int ni = 0; ni < 4; ni++)
#pragma unroll
                        for (int e = 0; e < 4; e++) d[mi][ni][e] = 0.f;
            }
            if (++s == kStages) { s = 0; parity ^= 1; }
            if (++j == kWSlots) { j = 0; wparity ^= 1; }
        }
        return;
    }
    {
        constexpr int LPR = CH > 0 ? CH / 4 : 32;  // lanes per feature row
        constexpr int G = 32 / LPR;                // lane groups sharing the 32 pixels
        constexpr int NQ = 8 / G;                  // 2x2 quads per lane
        const int b = warp - L::kFeatWarp0;
        const int grp = lane / LPR, cl = lane % LPR;
        // Accumulators [quad][pixel in quad][channel].  With F3DGS_FFMA2 the two pixels of a quad row share a 64-bit
        // register pair and one paired FMA (fma2_rn: feature channel broadcast x weight pair + accumulator pair) covers
        // both; each half is an IEEE fma.rn, so the results are bit-identical to the scalar loop.
#if F3DGS_FFMA2
        float2 acc2[NQ][2][4];  // [quad][pixel pair (row of the 2x2 quad)][channel]
#define ACC(q, i, c) (((i) & 1) ? acc2[q][(i) >> 1][c].y : acc2[q][(i) >> 1][c].x)
#else
        float acc[NQ][4][4];
#define ACC(q, i, c) acc[q][i][c]
#endif
#pragma unroll
        for (int q = 0; q < NQ; q++)
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int c = 0; c < 4; c++) ACC(q, i, c) = 0.f;
#define FEAT_ROW_FMA(Q, ROW, W2)                                                                     \
    do {                                                                                             \
        const float2 w2_ = (W2);                                                                     \
        const float fr_[4] = {f.x, f.y, f.z, f.w};                                                   \
        _Pragma("unroll") for (int c_ = 0; c_ < 4; c_++)                                             \
            acc2[Q][ROW][c_] = fma2_rn(make_float2(fr_[c_], fr_[c_]), w2_, acc2[Q][ROW][c_]);     \
    } while (0)
#if F3DGS_FFMA2
#define FEAT_QUAD_FMA(Q, W4)                                                                         \
    do {                                                                                             \
        const float2 w01_ = make_float2((W4).x, (W4).y), w23_ = make_float2((W4).z, (W4).w);         \
        const float fc_[4] = {f.x, f.y, f.z, f.w};                                                   \
        _Pragma("unroll") for (int c_ = 0; c_ < 4; c_++) {                                           \
            const float2 fb_ = make_float2(fc_[c_], fc_[c_]);                                        \
            acc2[Q][0][c_] = fma2_rn(fb_, w01_, acc2[Q][0][c_]);                                  \
            acc2[Q][1][c_] = fma2_rn(fb_, w23_, acc2[Q][1][c_]);                                  \
        }                                                                                            \
    } while (0)
#else
#define FEAT_QUAD_FMA(Q, W4)                                                                         \
    do {                                                                                             \
        const float wv_[4] = {(W4).x, (W4).y, (W4).z, (W4).w};                                       \
        _Pragma("unroll") for (int i_ = 0; i_ < 4; i_++) {                                           \
            acc[Q][i_][0] = fmaf(f.x, wv_[i_], acc[Q][i_][0]);                                       \
            acc[Q][i_][1] = fmaf(f.y, wv_[i_], acc[Q][i_][1]);                                       \
            acc[Q][i_][2] = fmaf(f.z, wv_[i_], acc[Q][i_][2]);                                       \
            acc[Q][i_][3] = fmaf(f.w, wv_[i_], acc[Q][i_][3]);                                       \
        }                                                                                            \
    } while (0)
#endif
        int s = 0, j = 0;
        uint32_t parity = 0, wparity = 0;
        long long tF_wfull = 0, tF_full = 0, tF_epi = 0, tF_total = TICK(), nF_k = 0;
        for (;;) {
            { const long long t_ = TICK(); mbar_wait(&ring.wfull[b][j], wparity); tF_wfull += TICK() - t_; }
            const WSlot& ws = ring.ws[b][j];
            const int work = ws.work;
            if (work < 0) break;
            uint32_t km = ws.km;
            const uint32_t last = ws.last;
            { const long long t_ = TICK(); mbar_wait(&ring.full[s], parity); tF_full += TICK() - t_; }  // feature rows landed
            nF_k += __popc(km);
            if (F3DGS_DIAG_NO_FMA) km = 0;
            const Stage<CH>& st = ring.stage[s];
            if (L::kPrefetchW) {
                // 184-register layout: dense over the block with every operand of an instance fetched before its
                // 128 FFMAs (the compiler barrier keeps the nine LDS.128 ahead of the FFMA stream), so the FMA pipe
                // sees one uninterrupted run per instance.  Pixels that skipped the instance carry w = 0.
                while (km) {
                    const int k = __ffs(km) - 1;
                    km &= km - 1;
                    const float4 f = *reinterpret_cast<const float4*>(&st.feat[k][cl * 4]);
                    float4 w4[NQ];
#pragma unroll
                    for (int qi = 0; qi < NQ; qi++)
                        w4[qi] = *reinterpret_cast<const float4*>(&ws.w[k][4 * (qi * G + grp)]);
                    asm volatile("" ::: "memory");
#pragma unroll
                    for (int qi = 0; qi < NQ; qi++) {
                        FEAT_QUAD_FMA(qi, w4[qi]);
                    }
                }
            } else {
#if F3DGS_FEAT_PREFETCH
                // the next instance's pixel mask and feature float4 are requested before this instance's FMAs, so their
                // LDS latency hides behind the FMA stream instead of heading every instance
                int kn = km ? __ffs(km) - 1 : 0;
                uint32_t pm_n = ws.pm[kn];
                float4 f_n = *reinterpret_cast<const float4*>(&st.feat[kn][cl * 4]);
                while (km) {
                    const int k = kn;
                    const uint32_t pm = pm_n;
                    const float4 f = f_n;
                    km &= km - 1;
                    kn = km ? __ffs(km) - 1 : k;
                    pm_n = ws.pm[kn];
                    f_n = *reinterpret_cast<const float4*>(&st.feat[kn][cl * 4]);
#else
                while (km) {
                    const int k = __ffs(km) - 1;
                    km &= km - 1;
                    const uint32_t pm = ws.pm[k];
                    const float4 f = *reinterpret_cast<const float4*>(&st.feat[k][cl * 4]);
#endif
#pragma unroll
                    for (int qi = 0; qi < NQ; qi++) {
                        const int q = qi * G + grp;
                        if ((pm >> (4 * q)) & 0xFu) {
                            const float4 w4 = *reinterpret_cast<const float4*>(&ws.w[k][4 * q]);
#if F3DGS_PAIR_SKIP && F3DGS_FFMA2
                            // a pixel that did not blend has w = 0 and adds +0: skipping its FMAs leaves every accumulator
                            // bit-identical (fma(f, +0, acc) == acc for finite f; acc is never -0 because it starts at +0)
                            if ((pm >> (4 * q)) & 0x3u) FEAT_ROW_FMA(qi, 0, make_float2(w4.x, w4.y));
                            if ((pm >> (4 * q)) & 0xCu) FEAT_ROW_FMA(qi, 1, make_float2(w4.z, w4.w));
#else
                            FEAT_QUAD_FMA(qi, w4);
#endif
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&ring.wempty[b][j]);
                mbar_arrive(&ring.empty[s]);
            }
            const long long tE_ = TICK();
            if (last) {
                // ---- epilogue of this work item: write the block's 32 pixels x CH channels, reset
                const int tile = work / args.pa.chunks, chunk = work - tile * args.pa.chunks;
                const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
                const int bx0 = tile_x * 16 + (b & 1) * 8, by0 = tile_y * 16 + (b >> 1) * 4;
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const int ch = chunk * CH + cl * 4 + c;
                    if (ch < C) {
                        float* plane = args.out_feature + (size_t)ch * HW;
                        if (G == 1 && (args.vec_store & 2) && bx0 + 8 <= W) {
                            // lane holds all 8 quads: one 256-bit store = a full 32-byte sector per 8-pixel row
#pragma unroll
                            for (int y = 0; y < 4; y++) {
                                const int yy = by0 + y;
                                if (yy >= H) continue;
                                const int qa = (y >> 1) * 4, i0 = (y & 1) * 2;
                                st_na_f8(plane + (size_t)yy * W + bx0,
                                         make_float4(ACC(qa % NQ, i0, c), ACC(qa % NQ, i0 + 1, c),
                                                     ACC((qa + 1) % NQ, i0, c), ACC((qa + 1) % NQ, i0 + 1, c)),
                                         make_float4(ACC((qa + 2) % NQ, i0, c), ACC((qa + 2) % NQ, i0 + 1, c),
                                                     ACC((qa + 3) % NQ, i0, c), ACC((qa + 3) % NQ, i0 + 1, c)));
                            }
                        } else if (G == 1 && (args.vec_store & 1)) {
                            // rows of 8 pixels -> two 128-bit stores per row
#pragma unroll
                            for (int y = 0; y < 4; y++) {
                                const int yy = by0 + y;
                                if (yy >= H) continue;
#pragma unroll
                                for (int half = 0; half < 2; half++) {
                                    const int xx = bx0 + half * 4;
                                    if (xx >= W) continue;
                                    const int qa = (y >> 1) * 4 + half * 2, i0 = (y & 1) * 2;
                                    const float4 v =
                                        make_float4(ACC(qa % NQ, i0, c), ACC(qa % NQ, i0 + 1, c),
                                                    ACC((qa + 1) % NQ, i0, c), ACC((qa + 1) % NQ, i0 + 1, c));
                                    st_na_f4(plane + (size_t)yy * W + xx, v);
                                }
                            }
                        } else {
#pragma unroll
                            for (int qi = 0; qi < NQ; qi++) {
                                const int q = qi * G + grp;
#pragma unroll
                                for (int i = 0; i < 4; i++) {
                                    const int xx = bx0 + (q & 3) * 2 + (i & 1), yy = by0 + (q >> 2) * 2 + (i >> 1);
                                    if (xx < W && yy < H) plane[(size_t)yy * W + xx] = ACC(qi, i, c);
                                }
                            }
                        }
                    }
                }
#pragma unroll
                for (int q = 0; q < NQ; q++)
#pragma unroll
                    for (int i = 0; i < 4; i++)
#pragma unroll
                        for (int c = 0; c < 4; c++) ACC(q, i, c) = 0.f;
            }
            tF_epi += TICK() - tE_;
            if (++s == kStages) { s = 0; parity ^= 1; }
            if (++j == kWSlots) { j = 0; wparity ^= 1; }
        }
        if (kTiming && args.dbg && lane == 0) {
            long long* d = args.dbg + (blockIdx.x * 32 + warp) * 8;
            d[0] = clock64() - tF_total; d[1] = tF_wfull; d[2] = tF_full; d[3] = tF_epi; d[4] = nF_k;
        }
    }
}

// Warp layout (see Layout<> in composite_common.cuh): 8 alpha warps x 1 block (BPA = 1).  The 4 x 2 layout is not
// instantiated.
template <int CH, int BPA, bool TC>
static cudaError_t launch_fwd_t(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                const SplatRec* rec, const float* features, const float* bg, float* final_T,
                                uint32_t* n_contrib, float* out_color, float* out_feature, float* out_depth,
                                int* work_counter, cudaStream_t s) {
    const size_t smem = sizeof(RingV2<CH>);
    // the opt-in to > 48 KB of dynamic shared memory is per device (context): remember it per device ordinal, so that one
    // process driving several GPUs works too
    static std::atomic<int> sms_of_device[64];  // zero-initialised; set once per device (idempotent)
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    if (sms_of_device[dev].load() == 0) {
        cudaError_t e = cudaFuncSetAttribute(composite_fwd_kernel<CH, BPA, TC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem);
        if (e != cudaSuccess) return e;
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sms_of_device[dev].store(n > 0 ? n : 132);
    }
    const int num_sms = sms_of_device[dev].load();
    FwdArgs a;
    a.pa.ranges = ranges; a.pa.point_list = point_list; a.pa.rec = rec;
    a.pa.features = CH > 0 ? features : nullptr;
    a.pa.n_contrib = nullptr;
    a.pa.work_counter = work_counter;
    a.pa.W = vp.W; a.pa.H = vp.H; a.pa.C = vp.C;
    a.pa.tiles_x = (int)vp.grid_x;
    a.pa.num_tiles = (int)(vp.grid_x * vp.grid_y);
    a.pa.chunks = CH > 0 ? (vp.C + CH - 1) / CH : 1;
    a.pa.use_bulk = (CH > 0 && vp.C % 4 == 0 && (reinterpret_cast<uintptr_t>(features) & 15) == 0) ? 1 : 0;
    a.bg = bg; a.final_T = final_T; a.n_contrib = n_contrib;
    a.out_color = out_color; a.out_feature = out_feature; a.out_depth = out_depth;
    a.vec_store = (vp.W % 4 == 0 && (reinterpret_cast<uintptr_t>(out_feature) & 15) == 0) ? 1 : 0;
    if (vp.W % 8 == 0 && (reinterpret_cast<uintptr_t>(out_feature) & 31) == 0) a.vec_store |= 2;
    cudaError_t e = cudaMemsetAsync(work_counter, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    const int grid = min(a.pa.num_tiles * a.pa.chunks, num_sms);
    static long long* dbg = nullptr;
    const bool timing = kTiming && getenv("F3DGS_TIMING") != nullptr;  // debug aid (timing builds only): per-role cycle breakdown on stderr
    if (timing && !dbg) cudaMalloc(&dbg, 256 * 32 * 8 * sizeof(long long));
    a.dbg = timing ? dbg : nullptr;
    if (timing) cudaMemsetAsync(dbg, 0, 256 * 32 * 8 * sizeof(long long), s);
    composite_fwd_kernel<CH, BPA, TC><<<grid, Layout<BPA>::kThreads, smem, s>>>(a);
    g_launches++;
    if (timing) {
        static long long host[256 * 32 * 8];
        cudaMemcpyAsync(host, dbg, sizeof(host), cudaMemcpyDeviceToHost, s);
        cudaStreamSynchronize(s);
        const int nA = Layout<BPA>::kAlphaWarps, f0 = Layout<BPA>::kFeatWarp0;
        double prod = 0, A[5] = {0, 0, 0, 0, 0}, F[5] = {0, 0, 0, 0, 0};
        for (int c = 0; c < grid; c++) {
            prod += host[(c * 32 + 0) * 8];
            for (int w = 0; w < nA; w++) for (int i = 0; i < 5; i++) A[i] += host[(c * 32 + kAlphaWarp0 + w) * 8 + i];
            for (int w = 0; w < 8; w++) for (int i = 0; i < 5; i++) F[i] += host[(c * 32 + f0 + w) * 8 + i];
        }
        fprintf(stderr, "[f3dgs timing fwd CH=%d BPA=%d] per-warp mean cycles: producer %.0f | alpha total %.0f wait_full %.0f wait_wempty %.0f stages %.0f hits %.0f | feature total %.0f wait_wfull %.0f wait_full %.0f epilogue %.0f k %.0f\n",
                CH, BPA, prod / grid, A[0] / (grid * nA), A[1] / (grid * nA), A[2] / (grid * nA), A[3] / (grid * nA), A[4] / (grid * nA),
                F[0] / (grid * 8), F[1] / (grid * 8), F[2] / (grid * 8), F[3] / (grid * 8), F[4] / (grid * 8));
    }
    return cudaGetLastError();
}

#define F3DGS_FWD_DISPATCH(CHV, TC)                                                                          \
    launch_fwd_t<CHV, 1, TC>(vp, ranges, point_list, rec, features, bg, final_T, n_contrib, out_color, out_feature, \
                         out_depth, work_counter, s)

cudaError_t launch_composite_fwd(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                 const SplatRec* rec, const float* features, const float* bg,
                                 float* final_T, uint32_t* n_contrib, float* out_color,
                                 float* out_feature, float* out_depth, int* work_counter, cudaStream_t s) {
    if (vp.C == 0) return F3DGS_FWD_DISPATCH(0, false);
    if (vp.C <= 32) return F3DGS_FWD_DISPATCH(32, false);
    if (vp.C <= 64) return F3DGS_FWD_DISPATCH(64, false);
    return F3DGS_FWD_DISPATCH(128, false);
}

// Preconditions checked by the caller (api.cu): C % 4 == 0 and a 16-byte aligned feature matrix (the feature rows arrive
// by bulk copies); every other shape takes launch_composite_fwd.
cudaError_t launch_composite_fwd_tc(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                    const SplatRec* rec, const float* features, const float* bg,
                                    float* final_T, uint32_t* n_contrib, float* out_color,
                                    float* out_feature, float* out_depth, int* work_counter, cudaStream_t s) {
    if (vp.C <= 64) return F3DGS_FWD_DISPATCH(64, true);
    return F3DGS_FWD_DISPATCH(128, true);
}

}  // namespace f3dgs
