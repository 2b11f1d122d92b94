// Forward tile composite: front-to-back alpha blend of RGB, depth and a C-wide feature vector.
// Reference: forward.cu:261-396 (renderCUDA<3>), semantics restated in SURVEY.md A.4.
//
// Per pixel the arithmetic that decides WHAT is blended (power, alpha, T, the 1/255 and 1e-4
// tests, n_contrib, final_T) and the RGB/depth accumulation are the reference's expressions
// compiled by the same compiler (see common.cuh), so those outputs are bit-identical.  The feature
// accumulation uses acc = fma(f, alpha*T, acc) instead of fma(T, alpha*f, acc): one rounding
// differs per term (<= 1 ulp of the term), which halves the FMA-pipe work of the hot loop.
//
// Roles (composite_common.cuh): producer + copy warp -> alpha warps -> feature warps, persistent over tiles.
//   alpha warp b   lane = pixel of block b.  For every staged instance whose footprint reaches
//                  the block: alpha, T update, RGB/depth accumulate; publishes w = alpha*T as a
//                  [instance][pixel] tile + a 32-bit "which pixels blended" mask per instance, and
//                  two instance masks: which instances blended a pixel of rows 0-1 / rows 2-3.
//   feature warps  a pair per block: warp (b, h) owns the 8x2 half of block b made of rows 2h and
//   (b, h)         2h+1 (quads 4h..4h+3, mask bits 16h..16h+15); lane = float4 of channels.  It walks
//                  the instances of its half's mask and does acc[pixel][4] += w[pixel] * f[4] for the
//                  pixels of its half that blended, one 2x2-pixel quad at a time: one broadcast LDS.128
//                  of the quad's weights feeds the FMAs of the quad rows that blended; the next
//                  instance's mask and feature float4 are loaded during this one's FMAs.  The half's 16
//                  pixels x 4 channels (= 64 accumulators per lane at CH = 128) live in registers.
//                  Every accumulator sees the same FMAs in the same order as with one warp per block
//                  (an instance a warp skips adds nothing to its pixels), so the map is bitwise the
//                  same.  Hopper has no paired FP32 FMA (fma2_rn is two FFMAs): with one warp per block
//                  the feature FMAs cost 0.50 ms of 2.67 ms at config 3; with the pair, issued on two
//                  sub-partitions and skipping the other half's entries, 0.15 ms of 2.32 ms (README).
// Channel counts above 128 are split into chunks of 128 (extra work items); chunk 0 also writes
// colour, depth, final_T and n_contrib.
//
// Feature element type TF (float or __half): the per-Gaussian features and the feature map share it.  A float16 ring
// stages half the bytes per row; the feature warps upcast each channel exactly as they load it, accumulate in float32
// exactly as for float32 features, and the epilogue rounds each accumulator once to nearest even.  So a float16 render
// is bitwise the float32 render of the upcast features followed by .half(), and everything else is bitwise the float32
// render's (the alpha warps never read features).
//
// PLANES (opt-in): the alpha warps also accumulate I = sum_i w_i (1/z_i) beside the depth, with 1/z_i the correctly
// rounded reciprocal of the record's view depth, and the epilogue writes the opacity plane 1 - T (the T that goes to
// final_T) and the inverse-depth plane I.  Nothing else the kernel computes or stores changes, so colour, depth, the
// feature map, final_T and n_contrib are bitwise those of the kernel without the planes.
//
// DIST (opt-in, not with PLANES): the alpha warps also accumulate the depth distortion loss
// L_p = sum_ij w_i w_j |z_i - z_j| = 2 sum_i w_i (z_i A_i - D_i), A_i = 1 - T_i, D_i = sum_{j<i} w_j z_j, with z_i the
// record's view depth.  The tile sort key orders each tile list by z, so this prefix-sum form is the pairwise sum.  Per
// blended pair Q += w (z (1 - T) - Dp) before Dp takes the pair, and the epilogue writes 2Q.  As with PLANES nothing else
// changes, so every other output is bitwise that of the kernel without it.
//
// Registers: with features the 28 warps are launched at 72 registers per thread (64512 in the CTA pool); setmaxnreg
// then gives the producer group 40, the alpha warps 56 and the feature warps 88 (4x32x40 + 8x32x56 + 16x32x88 =
// 64512).  (setmaxnreg acts per warpgroup of 4 consecutive warps, so the producer group is one unit.)  Without
// features the 20 warps are launched at 96, and the producer group gets 40 and the alpha warps 64.
#include <type_traits>

#include "composite_common.cuh"

namespace f3dgs {

// With features: the producer group, 8 alpha warps and 16 feature warps.  Without features the kernel keeps its
// 20-warp launch (the 8 warps after the alpha warps return at once).
template <int CH>
constexpr int kFwdThreads = (kFeatWarp0 + (CH > 0 ? 2 : 1) * kBlocksPerTile) * 32;
template <int CH>
constexpr int kRegsAlpha = CH > 0 ? 56 : 64;
constexpr int kRegsFeature = 88;

template <typename TF>
struct FwdArgs {
    ProducerArgs pa;
    const float* bg;
    float* final_T;
    uint32_t* n_contrib;
    float* out_color;
    TF* out_feature;
    float* out_depth;
    int vec_store;
    float* out_alpha;     // PLANES: [H,W] 1 - final_T
    float* out_invdepth;  // PLANES: [H,W] sum_i w_i / z_i
    float* out_distortion;  // DIST: [H,W] sum_ij w_i w_j |z_i - z_j|
};

// A lane's 4 channels of a staged feature row as loaded (float4, or 8 bytes of float16; to_float4 makes them float32).
template <typename TF>
using Feat4 = std::conditional_t<std::is_same_v<TF, float>, float4, uint2>;
// two accumulators rounded to float16 (nearest even, as torch's .half()), packed low = a
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
// Stores of the feature map in the three access shapes of for_tile_pixels: an 8-pixel row (a full 32-byte sector of
// float, 16 bytes of half), a 4-pixel run (16 / 8 bytes) and one pixel
__device__ __forceinline__ void st_row(float* p, float4 a, float4 b) { st_na_f8(p, a, b); }
__device__ __forceinline__ void st_row(__half* p, float4 a, float4 b) {
    st_na_b128(p, make_uint4(pack_half2(a.x, a.y), pack_half2(a.z, a.w), pack_half2(b.x, b.y), pack_half2(b.z, b.w)));
}
__device__ __forceinline__ void st_run(float* p, float4 v) { st_na_f4(p, v); }
__device__ __forceinline__ void st_run(__half* p, float4 v) {
    st_na_b64(p, make_uint2(pack_half2(v.x, v.y), pack_half2(v.z, v.w)));
}
__device__ __forceinline__ void st_px(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_px(__half* p, float v) { *p = __float2half_rn(v); }

template <int CH, typename TF, bool PLANES, bool DIST = false>
__global__ void __launch_bounds__(kFwdThreads<CH>, 1)
composite_fwd_kernel(const FwdArgs<TF> args) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using RING = RingV2<CH, TF>;
    RING& ring = *reinterpret_cast<RING*>(smem_raw);
    // The warp index goes through a shuffle so that ptxas knows it is warp-uniform: role branches, ring/slot addresses
    // and everything loaded from them (instance masks, work ids) then live in uniform registers, the per-quad branches
    // of the feature loop need no BSSY/BSYNC reconvergence pair, and nothing is re-derived from SR_TID inside the loops.
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const int lane = threadIdx.x & 31;
    const int W = args.pa.W, H = args.pa.H, C = args.pa.C;
    const size_t HW = (size_t)H * W;

    ring_init<CH>(ring, CH > 0 ? kAlphaWarps + 2 * kBlocksPerTile : kAlphaWarps, CH > 0 ? 2 : 1, CH > 0 ? 2 : 1);
    __syncthreads();

    // ======================================================================== producer group
    if (warp < kAlphaWarp0) {
        reg_dec<kRegsProducer>();
        if (warp == kProducerWarp) {
            producer_loop<CH, false>(ring, args.pa);
        } else if constexpr (CH > 0) {
            if (warp == kProducerWarp + 1) copy_loop<CH, TF>(ring, args.pa);
        }
        return;
    }

    // ======================================================================== alpha warps
    if (warp < kFeatWarp0) {
        reg_dec<kRegsAlpha<CH>>();
        const int b = warp - kAlphaWarp0;  // owns pixel block b
        int s = 0, j = 0;
        uint32_t parity = 0, wparity = 1;  // wempty: fresh barrier falls through on parity 1
        float T = 1.f, Cr = 0.f, Cg = 0.f, Cb = 0.f, Dp = 0.f, pxf = 0.f, pyf = 0.f, fbx0 = 0.f, fby0 = 0.f;
        float Ip = 0.f;  // PLANES
        float Q = 0.f;   // DIST: half the distortion so far
        uint32_t last_contrib = 0;
        int px = 0, py = 0, chunk = 0;
        bool done = true, inside = false, blk_done = true;
        ROLE_CLK(uint32_t clk_full = 0, clk_wempty = 0; const uint32_t clk_0 = (uint32_t)clock64();)
        for (;;) {
            ROLE_CLK_WAIT(clk_full, mbar_wait(&ring.full[s], parity));
            Stage<CH, TF>& st = ring.stage[s];
            const uint32_t n = st.n, last = st.last, first = st.first;
            const int work = st.work;
            if (work < 0) break;
            if (first) {
                const int tile = work / args.pa.chunks;
                chunk = work - tile * args.pa.chunks;
                const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
                const int bx0 = block_x0(tile_x, b), by0 = block_y0(tile_y, b);
                px = bx0 + slot_px(lane);
                py = by0 + slot_py(lane);
                inside = px < W && py < H;
                pxf = (float)px; pyf = (float)py;
                fbx0 = (float)bx0; fby0 = (float)by0;
                T = 1.f; Cr = Cg = Cb = Dp = 0.f;
                if constexpr (PLANES) Ip = 0.f;
                if constexpr (DIST) Q = 0.f;
                last_contrib = 0;
                done = !inside;
                blk_done = __all_sync(0xffffffffu, done);
                if (blk_done && lane == 0) atomicOr(&ring.done_mask[st.done_slot], 1u << b);
            }
            WSlot* ws = &ring.ws[b][j];
            if (CH > 0) ROLE_CLK_WAIT(clk_wempty, mbar_wait(&ring.wempty[b][j], wparity));
            uint32_t km0 = 0, km1 = 0;  // instances that blended a pixel of rows 0-1 / rows 2-3
            if (!blk_done && n > 0) {
                bool hit = false;
                if (lane < n) hit = footprint_hits_rect(st.rec0[lane], st.rec1[lane], fbx0, fbx0 + 7.f, fby0, fby0 + 3.f);
                uint32_t am = __ballot_sync(0xffffffffu, hit);
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
                    for (int u = 0; u < 4; u++) al[u] = splat_alpha(st.rec0[kk[u]], st.rec1[kk[u]], pxf, pyf, vk[u]).alpha;
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        if (!vk[u]) break;  // warp-uniform, only in the last trip
                        const float4 r2 = st.rec2[kk[u]];
                        const uint32_t lp = st.listpos[kk[u]];
                        const float alpha = al[u];
                        const float test_T = T * (1 - alpha);
                        const bool act = !done && alpha > 0.f;
                        const bool stop = act && (test_T < 0.0001f);  // reference: done = true, not blended
                        const bool blend = act && !stop;
                        done = done || stop;
                        const float wgt = blend ? alpha * T : 0.f;
                        const float nCr = Cr + r2.x * alpha * T;  // reference forward.cu:362-368
                        const float nCg = Cg + r2.y * alpha * T;
                        const float nCb = Cb + r2.z * alpha * T;
                        const float nDp = Dp + r2.w * (alpha * T);
                        if constexpr (DIST) {  // before Dp takes this pair: Dp = D_i, 1 - T = A_i
                            const float nQ = Q + (alpha * T) * (r2.w * (1.f - T) - Dp);
                            Q = blend ? nQ : Q;
                        }
                        Cr = blend ? nCr : Cr;
                        Cg = blend ? nCg : Cg;
                        Cb = blend ? nCb : Cb;
                        Dp = blend ? nDp : Dp;
                        if constexpr (PLANES) {
                            const float nIp = Ip + __frcp_rn(r2.w) * (alpha * T);
                            Ip = blend ? nIp : Ip;
                        }
                        T = blend ? test_T : T;
                        last_contrib = blend ? lp : last_contrib;
                        const uint32_t pm = __ballot_sync(0xffffffffu, blend);
                        if (CH > 0) {
                            ws->w[kk[u]][lane] = wgt;
                            if (lane == 0) ws->pm[kk[u]] = pm;
                            km0 |= ((pm & 0xFFFFu) ? 1u : 0u) << kk[u];
                            km1 |= ((pm >> 16) ? 1u : 0u) << kk[u];
                        }
                    }
                }
                if (__all_sync(0xffffffffu, done)) {
                    blk_done = true;
                    if (lane == 0) atomicOr(&ring.done_mask[st.done_slot], 1u << b);
                }
            }
            if (CH > 0) {
                __syncwarp();
                if (lane == 0) {
                    ws->km[0] = km0;
                    ws->km[1] = km1;
                    ws->last = last;
                    ws->first = first;
                    ws->work = work;
                    mbar_arrive(&ring.wfull[b][j]);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&ring.empty[s]);
            if (last && chunk == 0 && inside) {
                const size_t pix = (size_t)py * W + px;
                args.final_T[pix] = T;
                args.n_contrib[pix] = last_contrib;
                args.out_color[pix] = Cr + T * args.bg[0];  // reference forward.cu:389
                args.out_color[HW + pix] = Cg + T * args.bg[1];
                args.out_color[2 * HW + pix] = Cb + T * args.bg[2];
                args.out_depth[pix] = Dp;
                if constexpr (PLANES) {
                    args.out_alpha[pix] = 1.f - T;
                    args.out_invdepth[pix] = Ip;
                }
                if constexpr (DIST) args.out_distortion[pix] = 2.f * Q;
            }
            if (++s == kStages) { s = 0; parity ^= 1; }
            if (CH > 0 && ++j == kWSlots) { j = 0; wparity ^= 1; }
        }
        ROLE_CLK(if (lane == 0) {
            ROLE_CLK_ADD(kClkAlphaFull, clk_full);
            ROLE_CLK_ADD(kClkAlphaWempty, clk_wempty);
            ROLE_CLK_ADD(kClkAlphaLoop, (uint32_t)clock64() - clk_0);
        })
        if (CH > 0) {  // tell the feature warps of this block that the work is over
            mbar_wait(&ring.wempty[b][j], wparity);
            if (lane == 0) {
                ring.ws[b][j].work = -1;
                ring.ws[b][j].km[0] = ring.ws[b][j].km[1] = 0;
                mbar_arrive(&ring.wfull[b][j]);
            }
        }
        return;
    }

    // ======================================================================== feature warps
    if (CH == 0) return;
    reg_inc<kRegsFeature>();
    {  // own scope: ending the accumulators' lifetime here keeps the instruction schedule the kernel was tuned with
        constexpr int LPR = CH > 0 ? CH / 4 : 32;  // lanes per feature row
        constexpr int G = 32 / LPR;                // lane groups sharing the half's 16 pixels
        constexpr int NQ = 4 / G;                  // 2x2 quads of the warp's 8x2 half per lane
        // Warps kFeatWarp0 + 2b and + 2b + 1 are block b's pair.  Warp w runs on sub-partition w % 4, so each
        // sub-partition holds four feature warps: the upper halves (h = 0) of the even blocks on sub-partition 0, the
        // lower halves of the even blocks on 1, and the odd blocks' halves on 2 and 3.  The two halves of a block run on
        // different sub-partitions.
        const int b = (warp - kFeatWarp0) >> 1, h = (warp - kFeatWarp0) & 1;
        const int grp = lane / LPR, cl = lane % LPR;
        // Accumulators [quad][pixel pair (row of the 2x2 quad)][channel]: the two pixels of a quad row share a 64-bit register
        // pair and one paired FMA (fma2_rn: feature channel broadcast x weight pair + accumulator pair) covers both; each half
        // is an IEEE fma.rn, so the results are bit-identical to a scalar loop.
        float2 acc2[NQ][2][4];
#pragma unroll
        for (int q = 0; q < NQ; q++)
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int c = 0; c < 4; c++) tile_px(acc2, q, i, c) = 0.f;
#define FEAT_ROW_FMA(Q, ROW, W2)                                                                     \
        do {                                                                                             \
            const float2 w2_ = (W2);                                                                     \
            const float fr_[4] = {f.x, f.y, f.z, f.w};                                                   \
            _Pragma("unroll") for (int c_ = 0; c_ < 4; c_++)                                             \
                acc2[Q][ROW][c_] = fma2_rn(make_float2(fr_[c_], fr_[c_]), w2_, acc2[Q][ROW][c_]);     \
        } while (0)
        int s = 0, j = 0;
        uint32_t parity = 0, wparity = 0;
        ROLE_CLK(uint32_t clk_wfull = 0, clk_full = 0; const uint32_t clk_0 = (uint32_t)clock64();)
        for (;;) {
            ROLE_CLK_WAIT(clk_wfull, mbar_wait(&ring.wfull[b][j], wparity));
            const WSlot& ws = ring.ws[b][j];
            const int work = ws.work;
            if (work < 0) break;
            uint32_t km = ws.km[h];
            const uint32_t last = ws.last;
            ROLE_CLK_WAIT(clk_full, mbar_wait(&ring.full[s], parity));  // feature rows landed
            const Stage<CH, TF>& st = ring.stage[s];
            // the next instance's pixel mask and feature float4 are requested before this instance's FMAs, so their
            // LDS latency hides behind the FMA stream instead of heading every instance
            int kn = km ? __ffs(km) - 1 : 0;
            uint32_t pm_n = ws.pm[kn];
            Feat4<TF> f_n = *reinterpret_cast<const Feat4<TF>*>(&st.feat[kn][cl * 4]);
            while (km) {
                const int k = kn;
                const uint32_t pm = pm_n >> (16 * h);  // the half's pixels: quad q of the half in bits 4q..4q+3
                const float4 f = to_float4(f_n);
                km &= km - 1;
                kn = km ? __ffs(km) - 1 : k;
                pm_n = ws.pm[kn];
                f_n = *reinterpret_cast<const Feat4<TF>*>(&st.feat[kn][cl * 4]);
#pragma unroll
                for (int qi = 0; qi < NQ; qi++) {
                    const int q = qi * G + grp;
                    if ((pm >> (4 * q)) & 0xFu) {
                        const float4 w4 = *reinterpret_cast<const float4*>(&ws.w[k][16 * h + 4 * q]);
                        // a pixel that did not blend has w = 0 and adds +0: skipping its FMAs leaves every accumulator
                        // bit-identical (fma(f, +0, acc) == acc for finite f; acc is never -0 because it starts at +0)
                        if ((pm >> (4 * q)) & 0x3u) FEAT_ROW_FMA(qi, 0, make_float2(w4.x, w4.y));
                        if ((pm >> (4 * q)) & 0xCu) FEAT_ROW_FMA(qi, 1, make_float2(w4.z, w4.w));
                    }
                }
            }
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&ring.wempty[b][j]);
                mbar_arrive(&ring.empty[s]);
            }
            if (last) {
                // ---- epilogue of this work item: write the half's 16 pixels x CH channels, reset
                const int tile = work / args.pa.chunks, chunk = work - tile * args.pa.chunks;
                const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
                const int bx0 = block_x0(tile_x, b), by0 = block_y0(tile_y, b) + 2 * h;
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const int ch = chunk * CH + cl * 4 + c;
                    if (ch < C)
                        for_tile_pixels<G, NQ, 2>(
                            args.out_feature + (size_t)ch * HW, bx0, by0, W, H, grp, args.vec_store & 2,
                            args.vec_store & 1,
                            [&](TF* p, int y) { st_row(p, tile_run(acc2, y, 0, c), tile_run(acc2, y, 1, c)); },
                            [&](TF* p, int y, int half) { st_run(p, tile_run(acc2, y, half, c)); },
                            [&](TF* p, int qi, int i) { st_px(p, tile_px(acc2, qi, i, c)); });
                }
#pragma unroll
                for (int q = 0; q < NQ; q++)
#pragma unroll
                    for (int i = 0; i < 4; i++)
#pragma unroll
                        for (int c = 0; c < 4; c++) tile_px(acc2, q, i, c) = 0.f;
            }
            if (++s == kStages) { s = 0; parity ^= 1; }
            if (++j == kWSlots) { j = 0; wparity ^= 1; }
        }
        ROLE_CLK(if (lane == 0) {
            ROLE_CLK_ADD(kClkFeatWfull, clk_wfull);
            ROLE_CLK_ADD(kClkFeatFull, clk_full);
            ROLE_CLK_ADD(kClkFeatLoop, (uint32_t)clock64() - clk_0);
        })
    }
#undef FEAT_ROW_FMA
}

template <int CH, typename TF, bool PLANES, bool DIST = false>
static cudaError_t launch_fwd_t(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                const SplatRec* rec, const TF* features, const float* bg, float* final_T,
                                uint32_t* n_contrib, float* out_color, TF* out_feature, float* out_depth,
                                int* work_counter, cudaStream_t s, float* out_alpha, float* out_invdepth,
                                float* out_distortion) {
    const size_t smem = sizeof(RingV2<CH, TF>);
    int num_sms = 0;
    cudaError_t e = device_sms<composite_fwd_kernel<CH, TF, PLANES, DIST>>(num_sms, smem);
    if (e != cudaSuccess) return e;
    FwdArgs<TF> a;
    a.pa = producer_args(vp, ranges, point_list, rec, nullptr, work_counter);
    a.pa.features = CH > 0 ? features : nullptr;
    a.pa.C = vp.C;
    a.pa.chunks = CH > 0 ? (vp.C + CH - 1) / CH : 1;
    // bulk copies move rows of a multiple of 16 bytes from 16-byte aligned addresses: C % 4 == 0 (float), C % 8 == 0
    // (half)
    constexpr int kPer16 = 16 / (int)sizeof(TF);
    a.pa.use_bulk = (CH > 0 && vp.C % kPer16 == 0 && (reinterpret_cast<uintptr_t>(features) & 15) == 0) ? 1 : 0;
    a.bg = bg; a.final_T = final_T; a.n_contrib = n_contrib;
    a.out_color = out_color; a.out_feature = out_feature; a.out_depth = out_depth;
    a.out_alpha = out_alpha; a.out_invdepth = out_invdepth; a.out_distortion = out_distortion;
    // 1: 4-pixel stores (16 B of float, 8 B of half); 2: 8-pixel rows (32 B of float, 16 B of half)
    const uintptr_t out_addr = reinterpret_cast<uintptr_t>(out_feature);
    a.vec_store = (vp.W % 4 == 0 && (out_addr & (4 * sizeof(TF) - 1)) == 0) ? 1 : 0;
    if (vp.W % 8 == 0 && (out_addr & (8 * sizeof(TF) - 1)) == 0) a.vec_store |= 2;
    e = cudaMemsetAsync(work_counter, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    const int grid = min(a.pa.num_tiles * a.pa.chunks, num_sms);
    composite_fwd_kernel<CH, TF, PLANES, DIST><<<grid, kFwdThreads<CH>, smem, s>>>(a);
    g_launches++;
    return cudaGetLastError();
}

template <typename TF>
cudaError_t launch_composite_fwd(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                 const SplatRec* rec, const TF* features, const float* bg,
                                 float* final_T, uint32_t* n_contrib, float* out_color,
                                 TF* out_feature, float* out_depth, int* counters, cudaStream_t s, float* out_alpha,
                                 float* out_invdepth, float* out_distortion) {
    int* const work_counter = counters + kCounterFwd;
    if (vp.C == 0) {  // no feature rows or map: one kernel for both element types
        const auto launch0 = out_distortion ? launch_fwd_t<0, float, false, true>
                             : out_alpha    ? launch_fwd_t<0, float, true>
                                            : launch_fwd_t<0, float, false>;
        return launch0(vp, ranges, point_list, rec, nullptr, bg, final_T, n_contrib, out_color, nullptr, out_depth,
                       work_counter, s, out_alpha, out_invdepth, out_distortion);
    }
    const int ch = channel_chunk(vp.C);
    const auto launch = out_distortion ? (ch == 32   ? launch_fwd_t<32, TF, false, true>
                                          : ch == 64 ? launch_fwd_t<64, TF, false, true>
                                                     : launch_fwd_t<128, TF, false, true>)
                        : out_alpha    ? (ch == 32   ? launch_fwd_t<32, TF, true>
                                          : ch == 64 ? launch_fwd_t<64, TF, true>
                                                     : launch_fwd_t<128, TF, true>)
                                       : (ch == 32   ? launch_fwd_t<32, TF, false>
                                          : ch == 64 ? launch_fwd_t<64, TF, false>
                                                     : launch_fwd_t<128, TF, false>);
    return launch(vp, ranges, point_list, rec, features, bg, final_T, n_contrib, out_color, out_feature, out_depth,
                  work_counter, s, out_alpha, out_invdepth, out_distortion);
}

template cudaError_t launch_composite_fwd<float>(const ViewParams&, const uint2*, const uint32_t*, const SplatRec*,
                                                 const float*, const float*, float*, uint32_t*, float*, float*, float*,
                                                 int*, cudaStream_t, float*, float*, float*);
template cudaError_t launch_composite_fwd<__half>(const ViewParams&, const uint2*, const uint32_t*, const SplatRec*,
                                                  const __half*, const float*, float*, uint32_t*, float*, __half*,
                                                  float*, int*, cudaStream_t, float*, float*, float*);

}  // namespace f3dgs

#ifdef F3DGS_ROLE_CLOCKS
ROLE_CLK_EXPORT(f3dgs_role_clocks_fwd)
#endif
