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
//                  [instance][pixel] tile + a 32-bit "which pixels blended" mask per instance.
//   feature warp b lane = float4 of channels.  acc[pixel][4] += w[pixel] * f[4] for the pixels in
//                  the mask, one 2x2-pixel quad at a time: one broadcast LDS.128 of the quad's weights
//                  feeds paired FMAs on the quad rows that blended; the next instance's mask and feature
//                  float4 are loaded during this one's FMAs.  All 32 pixels x 4 channels (= 128
//                  accumulators per lane at CH = 128) live in registers.
// Channel counts above 128 are split into chunks of 128 (extra work items); chunk 0 also writes
// colour, depth, final_T and n_contrib.
//
// Feature element type TF (float or __half): the per-Gaussian features and the feature map share it.  A float16 ring
// stages half the bytes per row; the feature warps upcast each channel exactly as they load it, accumulate in float32
// exactly as for float32 features, and the epilogue rounds each accumulator once to nearest even.  So a float16 render
// is bitwise the float32 render of the upcast features followed by .half(), and everything else is bitwise the float32
// render's (the alpha warps never read features).
//
// Registers: the 20 warps are launched at 96 registers per thread (61440 in the CTA pool); setmaxnreg then gives the
// producer group 40, the alpha warps 64 and the feature warps 152 (4x32x40 + 8x32x64 + 8x32x152 = 60416).
#include <type_traits>

#include "composite_common.cuh"

namespace f3dgs {

constexpr int kFwdThreads = (kFeatWarp0 + kBlocksPerTile) * 32;
constexpr int kRegsAlpha = 64;
constexpr int kRegsFeature = 152;

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
};

// A lane's 4 channels of a staged feature row as loaded (float4, or 8 bytes of float16) and as float32 (exact).
template <typename TF>
using Feat4 = std::conditional_t<std::is_same_v<TF, float>, float4, uint2>;
__device__ __forceinline__ float4 feat_f32(float4 v) { return v; }
__device__ __forceinline__ float4 feat_f32(uint2 v) {
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
// two accumulators rounded to float16 (nearest even, as torch's .half()), packed low = a
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

template <int CH, typename TF>
__global__ void __launch_bounds__(kFwdThreads, 1)
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

    ring_init<CH>(ring, CH > 0 ? kAlphaWarps + kBlocksPerTile : kAlphaWarps, CH > 0 ? 2 : 1);
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
        reg_dec<kRegsAlpha>();
        const int b = warp - kAlphaWarp0;  // owns pixel block b
        int s = 0, j = 0;
        uint32_t parity = 0, wparity = 1;  // wempty: fresh barrier falls through on parity 1
        float T = 1.f, Cr = 0.f, Cg = 0.f, Cb = 0.f, Dp = 0.f, pxf = 0.f, pyf = 0.f, fbx0 = 0.f, fby0 = 0.f;
        uint32_t last_contrib = 0;
        int px = 0, py = 0, chunk = 0;
        bool done = true, inside = false, blk_done = true;
        for (;;) {
            mbar_wait(&ring.full[s], parity);
            Stage<CH, TF>& st = ring.stage[s];
            const uint32_t n = st.n, last = st.last, first = st.first;
            const int work = st.work;
            if (work < 0) break;
            if (first) {
                const int tile = work / args.pa.chunks;
                chunk = work - tile * args.pa.chunks;
                const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
                const int bx0 = tile_x * 16 + (b & 1) * 8, by0 = tile_y * 16 + (b >> 1) * 4;
                px = bx0 + lane_px(lane);
                py = by0 + lane_py(lane);
                inside = px < W && py < H;
                pxf = (float)px; pyf = (float)py;
                fbx0 = (float)bx0; fby0 = (float)by0;
                T = 1.f; Cr = Cg = Cb = Dp = 0.f;
                last_contrib = 0;
                done = !inside;
                blk_done = __all_sync(0xffffffffu, done);
                if (blk_done && lane == 0) atomicOr(&ring.done_mask[st.done_slot], 1u << b);
            }
            WSlot* ws = &ring.ws[b][j];
            if (CH > 0) mbar_wait(&ring.wempty[b][j], wparity);
            uint32_t km = 0;
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
                    for (int u = 0; u < 4; u++) {
                        const float4 r0 = st.rec0[kk[u]];
                        const float4 r1 = st.rec1[kk[u]];
                        // same expression trees as reference forward.cu:340-351 (see common.cuh)
                        const float dx = r0.x - pxf, dy = r0.y - pyf;
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
                        Cr = blend ? nCr : Cr;
                        Cg = blend ? nCg : Cg;
                        Cb = blend ? nCb : Cb;
                        Dp = blend ? nDp : Dp;
                        T = blend ? test_T : T;
                        last_contrib = blend ? lp : last_contrib;
                        const uint32_t pm = __ballot_sync(0xffffffffu, blend);
                        if (CH > 0) {
                            ws->w[kk[u]][lane] = wgt;
                            if (lane == 0) ws->pm[kk[u]] = pm;
                            km |= (pm ? 1u : 0u) << kk[u];
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
                    ws->km = km;
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
            }
            if (++s == kStages) { s = 0; parity ^= 1; }
            if (CH > 0 && ++j == kWSlots) { j = 0; wparity ^= 1; }
        }
        if (CH > 0) {  // tell the feature warp of this block that the work is over
            mbar_wait(&ring.wempty[b][j], wparity);
            if (lane == 0) {
                ring.ws[b][j].work = -1;
                ring.ws[b][j].km = 0;
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
        constexpr int G = 32 / LPR;                // lane groups sharing the 32 pixels
        constexpr int NQ = 8 / G;                  // 2x2 quads per lane
        const int b = warp - kFeatWarp0;
        const int grp = lane / LPR, cl = lane % LPR;
        // Accumulators [quad][pixel pair (row of the 2x2 quad)][channel]: the two pixels of a quad row share a 64-bit register
        // pair and one paired FMA (fma2_rn: feature channel broadcast x weight pair + accumulator pair) covers both; each half
        // is an IEEE fma.rn, so the results are bit-identical to a scalar loop.
        float2 acc2[NQ][2][4];
#define ACC(q, i, c) (((i) & 1) ? acc2[q][(i) >> 1][c].y : acc2[q][(i) >> 1][c].x)
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
        int s = 0, j = 0;
        uint32_t parity = 0, wparity = 0;
        for (;;) {
            mbar_wait(&ring.wfull[b][j], wparity);
            const WSlot& ws = ring.ws[b][j];
            const int work = ws.work;
            if (work < 0) break;
            uint32_t km = ws.km;
            const uint32_t last = ws.last;
            mbar_wait(&ring.full[s], parity);  // feature rows landed
            const Stage<CH, TF>& st = ring.stage[s];
            // the next instance's pixel mask and feature float4 are requested before this instance's FMAs, so their
            // LDS latency hides behind the FMA stream instead of heading every instance
            int kn = km ? __ffs(km) - 1 : 0;
            uint32_t pm_n = ws.pm[kn];
            Feat4<TF> f_n = *reinterpret_cast<const Feat4<TF>*>(&st.feat[kn][cl * 4]);
            while (km) {
                const int k = kn;
                const uint32_t pm = pm_n;
                const float4 f = feat_f32(f_n);
                km &= km - 1;
                kn = km ? __ffs(km) - 1 : k;
                pm_n = ws.pm[kn];
                f_n = *reinterpret_cast<const Feat4<TF>*>(&st.feat[kn][cl * 4]);
#pragma unroll
                for (int qi = 0; qi < NQ; qi++) {
                    const int q = qi * G + grp;
                    if ((pm >> (4 * q)) & 0xFu) {
                        const float4 w4 = *reinterpret_cast<const float4*>(&ws.w[k][4 * q]);
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
                // ---- epilogue of this work item: write the block's 32 pixels x CH channels, reset
                const int tile = work / args.pa.chunks, chunk = work - tile * args.pa.chunks;
                const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
                const int bx0 = tile_x * 16 + (b & 1) * 8, by0 = tile_y * 16 + (b >> 1) * 4;
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const int ch = chunk * CH + cl * 4 + c;
                    if (ch < C) {
                        if constexpr (std::is_same_v<TF, float>) {
                            float* plane = args.out_feature + (size_t)ch * HW;
                            if (G == 1 && (args.vec_store & 2) && bx0 + 8 <= W) {
                                // lane holds all 8 quads: a full 32-byte sector per 8-pixel row
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
                        } else {
                            __half* plane = args.out_feature + (size_t)ch * HW;
                            if (G == 1 && (args.vec_store & 2) && bx0 + 8 <= W) {
                                // lane holds all 8 quads: one 16-byte store per 8-pixel row
#pragma unroll
                                for (int y = 0; y < 4; y++) {
                                    const int yy = by0 + y;
                                    if (yy >= H) continue;
                                    const int qa = (y >> 1) * 4, i0 = (y & 1) * 2;
                                    uint32_t h[4];
#pragma unroll
                                    for (int k = 0; k < 4; k++)
                                        h[k] = pack_half2(ACC((qa + k) % NQ, i0, c), ACC((qa + k) % NQ, i0 + 1, c));
                                    st_na_b128(plane + (size_t)yy * W + bx0, make_uint4(h[0], h[1], h[2], h[3]));
                                }
                            } else if (G == 1 && (args.vec_store & 1)) {
                                // rows of 8 pixels -> two 8-byte stores per row
#pragma unroll
                                for (int y = 0; y < 4; y++) {
                                    const int yy = by0 + y;
                                    if (yy >= H) continue;
#pragma unroll
                                    for (int half = 0; half < 2; half++) {
                                        const int xx = bx0 + half * 4;
                                        if (xx >= W) continue;
                                        const int qa = (y >> 1) * 4 + half * 2, i0 = (y & 1) * 2;
                                        const uint32_t h0 = pack_half2(ACC(qa % NQ, i0, c), ACC(qa % NQ, i0 + 1, c));
                                        const uint32_t h1 =
                                            pack_half2(ACC((qa + 1) % NQ, i0, c), ACC((qa + 1) % NQ, i0 + 1, c));
                                        st_na_b64(plane + (size_t)yy * W + xx, make_uint2(h0, h1));
                                    }
                                }
                            } else {
#pragma unroll
                                for (int qi = 0; qi < NQ; qi++) {
                                    const int q = qi * G + grp;
#pragma unroll
                                    for (int i = 0; i < 4; i++) {
                                        const int xx = bx0 + (q & 3) * 2 + (i & 1), yy = by0 + (q >> 2) * 2 + (i >> 1);
                                        if (xx < W && yy < H)
                                            plane[(size_t)yy * W + xx] = __float2half_rn(ACC(qi, i, c));
                                    }
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
            if (++s == kStages) { s = 0; parity ^= 1; }
            if (++j == kWSlots) { j = 0; wparity ^= 1; }
        }
    }
#undef FEAT_ROW_FMA
#undef ACC
}

template <int CH, typename TF>
static cudaError_t launch_fwd_t(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                const SplatRec* rec, const TF* features, const float* bg, float* final_T,
                                uint32_t* n_contrib, float* out_color, TF* out_feature, float* out_depth,
                                int* work_counter, cudaStream_t s) {
    const size_t smem = sizeof(RingV2<CH, TF>);
    // the opt-in to > 48 KB of dynamic shared memory is per device (context): remember it per device ordinal, so that one
    // process driving several GPUs works too
    static std::atomic<int> sms_of_device[64];  // zero-initialised; set once per device (idempotent)
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    if (sms_of_device[dev].load() == 0) {
        cudaError_t e = cudaFuncSetAttribute(composite_fwd_kernel<CH, TF>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sms_of_device[dev].store(n > 0 ? n : 132);
    }
    const int num_sms = sms_of_device[dev].load();
    FwdArgs<TF> a;
    a.pa.ranges = ranges; a.pa.point_list = point_list; a.pa.rec = rec;
    a.pa.features = CH > 0 ? features : nullptr;
    a.pa.n_contrib = nullptr;
    a.pa.work_counter = work_counter;
    a.pa.W = vp.W; a.pa.H = vp.H; a.pa.C = vp.C;
    a.pa.tiles_x = (int)vp.grid_x;
    a.pa.num_tiles = (int)(vp.grid_x * vp.grid_y);
    a.pa.chunks = CH > 0 ? (vp.C + CH - 1) / CH : 1;
    // bulk copies move rows of a multiple of 16 bytes from 16-byte aligned addresses: C % 4 == 0 (float), C % 8 == 0
    // (half)
    constexpr int kPer16 = 16 / (int)sizeof(TF);
    a.pa.use_bulk = (CH > 0 && vp.C % kPer16 == 0 && (reinterpret_cast<uintptr_t>(features) & 15) == 0) ? 1 : 0;
    a.bg = bg; a.final_T = final_T; a.n_contrib = n_contrib;
    a.out_color = out_color; a.out_feature = out_feature; a.out_depth = out_depth;
    // 1: 4-pixel stores (16 B of float, 8 B of half); 2: 8-pixel rows (32 B of float, 16 B of half)
    const uintptr_t out_addr = reinterpret_cast<uintptr_t>(out_feature);
    a.vec_store = (vp.W % 4 == 0 && (out_addr & (4 * sizeof(TF) - 1)) == 0) ? 1 : 0;
    if (vp.W % 8 == 0 && (out_addr & (8 * sizeof(TF) - 1)) == 0) a.vec_store |= 2;
    cudaError_t e = cudaMemsetAsync(work_counter, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    const int grid = min(a.pa.num_tiles * a.pa.chunks, num_sms);
    composite_fwd_kernel<CH, TF><<<grid, kFwdThreads, smem, s>>>(a);
    g_launches++;
    return cudaGetLastError();
}

template <typename TF>
cudaError_t launch_composite_fwd(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                 const SplatRec* rec, const TF* features, const float* bg,
                                 float* final_T, uint32_t* n_contrib, float* out_color,
                                 TF* out_feature, float* out_depth, int* work_counter, cudaStream_t s) {
    if (vp.C == 0)  // no feature rows or map: one kernel for both element types
        return launch_fwd_t<0, float>(vp, ranges, point_list, rec, nullptr, bg, final_T, n_contrib, out_color, nullptr,
                                      out_depth, work_counter, s);
    const auto launch = vp.C <= 32 ? launch_fwd_t<32, TF> : vp.C <= 64 ? launch_fwd_t<64, TF> : launch_fwd_t<128, TF>;
    return launch(vp, ranges, point_list, rec, features, bg, final_T, n_contrib, out_color, out_feature, out_depth,
                  work_counter, s);
}

template cudaError_t launch_composite_fwd<float>(const ViewParams&, const uint2*, const uint32_t*, const SplatRec*,
                                                 const float*, const float*, float*, uint32_t*, float*, float*, float*,
                                                 int*, cudaStream_t);
template cudaError_t launch_composite_fwd<__half>(const ViewParams&, const uint2*, const uint32_t*, const SplatRec*,
                                                  const __half*, const float*, float*, uint32_t*, float*, __half*,
                                                  float*, int*, cudaStream_t);

}  // namespace f3dgs
