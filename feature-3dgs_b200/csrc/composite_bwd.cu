// Backward tile composite, geometry kernel: walks each tile's instance list back to front and produces the per-Gaussian
// gradients of colour, depth, opacity, conic and 2-D mean.  The feature gradient is a second kernel (feature_bwd.cu)
// over the blend weights this one emits.
// Reference: backward.cu:407-620 (renderCUDA<3>), semantics restated in SURVEY.md A.5 / D.1.
//
// The reference issues (C+10) same-address global atomics per blended (pixel, Gaussian) pair.
// Here (roles as in composite_common.cuh, persistent over tiles; the producer group and the alpha warps only):
//   alpha warp a   lane = pixel of block a: recomputes alpha, unwinds T, and forms the 10 scalar gradient terms of the
//       pair (2-D mean x2, conic x3, opacity, depth, colour x3).  Lanes park their terms in a
//       [value][instance slot][pixel] shared tile; when 8 instances are parked the tile is summed row-wise (one lane per
//       row, conflict-free padded rows) and each row sum becomes ONE red.global.add -> 32x fewer atomics, none contended
//       inside the warp.
//   EMIT           with features, the alpha warps also append one list entry per (tile, block, instance that blended in
//       the block): {Gaussian id, pixel mask} + the 32 blend weights w = alpha*T, for feature_bwd.cu.
//   LIFT           feature lifting: the EMIT lists, and instead of the 10 gradient terms the one value w = alpha*T per pair,
//       reduced into weight_sum[P] through the same tile; no upstream gradient or background is read.  feature_bwd.cu
//       then forms sum_p w * map[:, p] over the lists with the teacher map in place of dL/dfeature_map.
//   SCORE          per-Gaussian scores of the view: LIFT's weights without the lists, three values per pair (w, 1, w)
//       parked in the same tile; the flush adds the first row sum into weight_sum, the second (a count of 0/1 floats,
//       at most 32 per row, exact) into pixel_count with an integer atomic, and takes the third row's max into
//       max_weight with an integer atomicMax on the float bits (w > 0, so the bits order as the floats do).
//   FEAT           the feature term of dL/dalpha (opt-in, after EMIT and feature_bwd): feature_dot (feature_bwd.cu) has
//       replaced each list entry's weights by the pair dot products d_ip = f_i . dL/dF_p; this walk repeats EMIT's, so a
//       pair's entry is the one EMIT wrote for it, and runs the colour term's scalar recurrence on d (no background:
//       the feature map has none), reducing the six geometric values into the same dL_dmean2D / dL_dconic / dL_dopacity.
//   PLANES         (GEOM and EMIT, opt-in) the gradients gA = dL/dA_p and gI = dL/dI_p of the forward's opacity plane
//       A_p = 1 - T_final and inverse-depth plane I_p = sum_i w_i / z_i.  dA/dalpha_i = T_final / (1 - alpha_i) is the
//       background term's factor, so gA joins it as bg.dL/dpix - gA; I gets the depth term's recurrence with 1/z_i in
//       place of z_i (dL/dI_p and one more float per lane), and dL/dz_i gains -w_i gI / z_i^2 in the same reduced value.
//       The walk reads only what every forward stores (records, final_T, n_contrib), and with gA = gI = 0 each added
//       term is an exact zero, so every output is bitwise that of the walk without PLANES.
// 12 warps and a ring without weight slots (RingSlim, 113 KB of shared memory with the reduction tiles): two CTAs per SM,
// and the alpha warps keep the launch register count (80).
// As in the reference, the feature loss does not feed dL/dalpha (backward.cu:575 is disabled) unless FEAT is asked for.
#include <mutex>

#include "composite_common.cuh"

namespace f3dgs {

constexpr int kBwdThreads = (kAlphaWarp0 + kAlphaWarps) * 32;
constexpr int kSlimCtas = 2;    // CTAs per SM
constexpr int kRedSlots = 8;
constexpr int kRedVals = 10;
constexpr int kRedRows = kRedSlots * kRedVals;
constexpr int kRedStride = 36;  // floats per row: lanes park at [row][lane] (conflict-free), rows are summed with
                                // LDS.128 (quarter-warp wavefronts: rows r..r+7 start 4 banks apart -> conflict-free)

struct alignas(128) BwdSmem {
    RingSlim ring;
    float red[kBlocksPerTile][kRedRows][kRedStride];
    uint32_t red_gid[kBlocksPerTile][kRedSlots];
};
static_assert(sizeof(BwdSmem) == 115200, "shared-memory layout changed");

struct BwdArgs {
    ProducerArgs pa;
    const float* bg;
    const float* final_T;
    const uint32_t* n_contrib;
    const float* dL_dpix;
    const float* dL_ddepth;
    float* dL_dmean2D;   // [P,3]
    float* dL_dconic;    // [P,4]
    float* dL_dopacity;  // [P]
    float* dL_dcolor;    // [P,3]
    float* dL_dz;        // [P]
    InstanceLists lists;  // EMIT and LIFT; w = alpha * T with the backward's unwound T.  FEAT: w = d_ip, read only
    float* weight_sum;    // LIFT: [P] += sum over the view's pixels of w
    const float* dL_dalpha;     // PLANES: [H,W] gA
    const float* dL_dinvdepth;  // PLANES: [H,W] gI
    float* max_weight;          // SCORE: [P] = max(max_weight, the largest w of the view)
    int64_t* pixel_count;       // SCORE: [P] += the number of pixels the Gaussian blended into
};

// GEOM: geometric gradients; EMIT: and the feature lists; LIFT: the feature lists and the per-Gaussian weight sums;
// FEAT: the feature term of the geometric gradients, from the lists' pair dot products; SCORE: LIFT's weights without
// the lists, reduced into the per-Gaussian weight sum, largest weight and blended-pixel count
enum class BwdMode { GEOM, EMIT, LIFT, FEAT, SCORE };
// Namespace-scope constants: as constexpr locals of the kernel they changed the register allocation of the EMIT
// instantiation, which is meant to stay instruction-for-instruction what it was before lifting existed.
template <BwdMode M>
constexpr bool kLift = M == BwdMode::LIFT;
template <BwdMode M>
constexpr bool kFeat = M == BwdMode::FEAT;
template <BwdMode M>
constexpr bool kScore = M == BwdMode::SCORE;
template <BwdMode M>  // values reduced per pair: FEAT has no depth or colour, SCORE reduces w, 1 and w
constexpr int kVals = kLift<M> ? 1 : (kFeat<M> ? 6 : (kScore<M> ? 3 : kRedVals));

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

// SCORE: one parked row of Gaussian gid (32 lanes, 0 where the pair did not blend) into its score v: 0 the weight sum,
// 1 the blended-pixel count, 2 the largest weight
__device__ __forceinline__ void score_flush_row(const BwdArgs& args, int v, uint32_t gid, const float* r) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f, m = 0.f;
    const float4* row = reinterpret_cast<const float4*>(r);
#pragma unroll
    for (int jj = 0; jj < 8; jj++) {
        const float4 q = row[jj];
        s0 += q.x;
        s1 += q.y;
        s2 += q.z;
        s3 += q.w;
        m = fmaxf(m, fmaxf(fmaxf(q.x, q.y), fmaxf(q.z, q.w)));
    }
    if (v == 0)
        red_add_f1(args.weight_sum + gid, (s0 + s1) + (s2 + s3));
    else if (v == 1)
        atomicAdd(reinterpret_cast<unsigned long long*>(args.pixel_count + gid),
                  (unsigned long long)((s0 + s1) + (s2 + s3)));
    else
        atomicMax(reinterpret_cast<int*>(args.max_weight + gid), __float_as_int(m));
}

template <BwdMode MODE, bool PLANES = false>
__global__ void __launch_bounds__(kBwdThreads, kSlimCtas)
composite_bwd_kernel(const BwdArgs args) {
    constexpr bool EMIT = MODE != BwdMode::GEOM && MODE != BwdMode::SCORE;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    BwdSmem& sm = *reinterpret_cast<BwdSmem*>(smem_raw);
    RingSlim& ring = sm.ring;
    // The warp index goes through a shuffle so that ptxas knows it is warp-uniform: role branches and ring addresses
    // then live in uniform registers, and nothing is re-derived from SR_TID inside the loops.
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const int lane = threadIdx.x & 31;
    const int W = args.pa.W, H = args.pa.H;
    const size_t HW = (size_t)H * W;

    ring_init<0>(ring, kAlphaWarps);
    __syncthreads();

    // ======================================================================== producer group
    if (warp < kAlphaWarp0) {
        reg_dec<kRegsProducer>();
        if (warp == kProducerWarp) producer_loop<0, true, RingSlim>(ring, args.pa);
        return;
    }

    // ======================================================================== alpha warps
    if (warp >= kAlphaWarp0 + kAlphaWarps) return;
    const int a = warp - kAlphaWarp0;  // owns pixel block a
    float(*red)[kRedStride] = sm.red[a];
    uint32_t* red_gid = sm.red_gid[a];
    uint32_t nslots = 0;  // warp-uniform
    int s = 0;
    uint32_t parity = 0;
    struct Px {
        float T, T_final, pxf, pyf, fbx0, fby0, dLp0, dLp1, dLp2, dLd, bg_dot;
        float ar0, ar1, ar2, lc0, lc1, lc2, last_alpha, accum_depth, last_depth;
        float gI, accum_invd;  // PLANES: dL/dI_p, and the 1/z recurrence's value for the pair the walk reaches next
        uint32_t last_contrib, wmax;
        bool inside;
    } p = Px{};
    size_t ebase = 0;     // EMIT: first list entry of this (tile, block)
    uint32_t ecount = 0;  // EMIT: entries written so far
    int etile = 0;
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;

    auto flush = [&]() {
        __syncwarp();
        for (int r = lane; r < kVals<MODE> * kRedSlots; r += 32) {
            const int slot = r % kRedSlots, v = r / kRedSlots;
            if constexpr (kScore<MODE>) {
                if (slot < (int)nslots) score_flush_row(args, v, red_gid[slot], red[r]);
            } else if (slot < (int)nslots) {
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
                if constexpr (kLift<MODE>)
                    red_add_f1(args.weight_sum + red_gid[slot], (s0 + s1) + (s2 + s3));
                else
                    red_add_f1(geom_dst(args, v, red_gid[slot]), (s0 + s1) + (s2 + s3));
            }
        }
        __syncwarp();
        nslots = 0;
    };

    ROLE_CLK(uint32_t clk_full = 0; const uint32_t clk_0 = (uint32_t)clock64();)
    for (;;) {
        ROLE_CLK_WAIT(clk_full, mbar_wait(&ring.full[s], parity));
        Stage<0>& st = ring.stage[s];
        const uint32_t n = st.n, last = st.last, first = st.first;
        const int work = st.work;
        if (work < 0) break;
        if (first) {
            const int tile = work / args.pa.chunks;
            const int tile_x = tile % args.pa.tiles_x, tile_y = tile / args.pa.tiles_x;
            if (EMIT) {
                etile = tile;
                const uint2 rg = args.pa.ranges[tile];
                ebase = list_begin(rg.x, rg.y, a);
                ecount = 0;
            }
            const int bx0 = block_x0(tile_x, a), by0 = block_y0(tile_y, a);
            const int px = bx0 + slot_px(lane), py = by0 + slot_py(lane);
            p.inside = px < W && py < H;
            p.pxf = (float)px; p.pyf = (float)py; p.fbx0 = (float)bx0; p.fby0 = (float)by0;
            const size_t pix = p.inside ? (size_t)py * W + px : 0;
            p.T_final = p.inside ? args.final_T[pix] : 0.f;
            p.T = p.T_final;
            p.last_contrib = p.inside ? args.n_contrib[pix] : 0u;
            p.dLp0 = p.dLp1 = p.dLp2 = p.dLd = 0.f;
            if constexpr (!kLift<MODE> && !kFeat<MODE> && !kScore<MODE>) {
                if (p.inside) {
                    p.dLp0 = args.dL_dpix[pix];
                    p.dLp1 = args.dL_dpix[HW + pix];
                    p.dLp2 = args.dL_dpix[2 * HW + pix];
                    p.dLd = args.dL_ddepth[pix];
                }
                p.bg_dot = args.bg[0] * p.dLp0 + args.bg[1] * p.dLp1 + args.bg[2] * p.dLp2;
                if constexpr (PLANES) {
                    p.gI = p.inside ? args.dL_dinvdepth[pix] : 0.f;
                    p.bg_dot -= p.inside ? args.dL_dalpha[pix] : 0.f;
                    p.accum_invd = 0.f;
                }
            }
            p.ar0 = p.ar1 = p.ar2 = p.lc0 = p.lc1 = p.lc2 = 0.f;
            p.last_alpha = p.accum_depth = p.last_depth = 0.f;
            uint32_t wm = p.last_contrib;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) wm = max(wm, __shfl_xor_sync(0xffffffffu, wm, o));
            p.wmax = wm;
        }
        if (n > 0 && p.wmax > 0) {
            bool hit = false;
            if (lane < n)
                hit = (st.listpos[lane] <= p.wmax) &&
                      footprint_hits_rect(st.rec0[lane], st.rec1[lane], p.fbx0, p.fbx0 + 7.f, p.fby0, p.fby0 + 3.f);
            uint32_t am = __ballot_sync(0xffffffffu, hit);
            while (am) {
                // branch-free evaluation of two instances per trip (see composite_fwd.cu)
                int kk[2];
                bool vk[2];
                SplatAlpha sa[2];
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    vk[u] = am != 0;
                    kk[u] = vk[u] ? (__ffs(am) - 1) : 0;
                    am &= am - 1;
                }
#pragma unroll
                for (int u = 0; u < 2; u++) sa[u] = splat_alpha(st.rec0[kk[u]], st.rec1[kk[u]], p.pxf, p.pyf, vk[u]);
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    if (!vk[u]) break;  // warp-uniform, only in the last trip
                    const int k = kk[u];
                    const float alpha = sa[u].alpha;
                    const bool contrib = p.inside && alpha > 0.f && st.listpos[k] <= p.last_contrib;
                    float wgt = 0.f;
                    float v[kRedVals];
#pragma unroll
                    for (int i = 0; i < kRedVals; i++) v[i] = 0.f;
                    if constexpr (kLift<MODE> || kScore<MODE>) {
                        if (contrib) {  // the T unwind below, without the gradient terms
                            p.T = p.T * rcp_approx(1.f - alpha);
                            wgt = alpha * p.T;
                            v[0] = wgt;
                            if constexpr (kScore<MODE>) {
                                v[1] = 1.f;
                                v[2] = wgt;
                            }
                        }
                    } else if constexpr (kFeat<MODE>) {
                        if (contrib) {  // the colour term below with the one channel d_ip and no background
                            const float d = args.lists.w[(ebase + ecount) * 32 + lane];
                            const float4 r1 = st.rec1[k];
                            p.T = p.T * rcp_approx(1.f - alpha);
                            p.ar0 = p.last_alpha * p.lc0 + (1.f - p.last_alpha) * p.ar0; p.lc0 = d;
                            const float dL_dalpha = (d - p.ar0) * p.T;
                            p.last_alpha = alpha;
                            const float Gs = sa[u].G, dx = sa[u].dx, dy = sa[u].dy;
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
                        }
                    } else if (contrib) {
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
                        float dLdz = p.dLd;
                        if constexpr (PLANES) {
                            // the depth term's recurrence with 1/z, advanced right away (the depth term advances it
                            // at the next pair, from last_alpha and last_depth): one register fewer
                            const float rz = __frcp_rn(r2.w);
                            dL_dalpha += (rz - p.accum_invd) * p.gI;
                            p.accum_invd = alpha * rz + (1.f - alpha) * p.accum_invd;
                            dLdz -= p.gI * (rz * rz);  // dI/dz_i = -w_i / z_i^2
                        }
                        dL_dalpha *= p.T;
                        p.last_alpha = alpha;
                        dL_dalpha += (-p.T_final * inv_1ma) * p.bg_dot;
                        const float Gs = sa[u].G, dx = sa[u].dx, dy = sa[u].dy;
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
                        v[6] = wgt * dLdz;
                    }
                    const uint32_t pm = __ballot_sync(0xffffffffu, contrib);
                    if (pm) {
                        if constexpr (kFeat<MODE>) {
#ifdef F3DGS_DEBUG_LISTS  // build.py's build_all(defines=("F3DGS_DEBUG_LISTS",)): the walks pair up
                            const uint2 m = args.lists.meta[ebase + ecount];
                            assert(m.x == st.gid[k] && m.y == pm);
#endif
                            ecount++;
                        } else if (EMIT) {  // one 128-byte row of weights + {id, mask} per blended (block, instance)
                            const size_t e = ebase + ecount;
                            args.lists.w[e * 32 + lane] = wgt;
                            if (lane == 0) args.lists.meta[e] = make_uint2(st.gid[k], pm);
                            ecount++;
                        }
#pragma unroll
                        for (int i = 0; i < kVals<MODE>; i++) red[i * kRedSlots + nslots][lane] = v[i];
                        if (lane == 0) red_gid[nslots] = st.gid[k];
                        nslots++;
                        if (nslots == kRedSlots) flush();
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&ring.empty[s]);
        if (EMIT && !kFeat<MODE> && last && lane == 0) args.lists.cnt[(size_t)etile * kBlocksPerTile + a] = ecount;
        if (last && nslots > 0) flush();
        if (++s == kStages) { s = 0; parity ^= 1; }
    }
    ROLE_CLK(if (lane == 0) {
        ROLE_CLK_ADD(kClkAlphaFull, clk_full);
        ROLE_CLK_ADD(kClkAlphaLoop, (uint32_t)clock64() - clk_0);
    })
}

// Stream-ordered scratch for the instance lists (the reference's backward allocates its scratch too,
// rasterizer_impl.cu:402-430); the default pool keeps freed blocks, so steady-state calls do not reach the driver.
// The caller releases *mem with cudaFreeAsync on the same stream.
static cudaError_t alloc_lists(size_t R, size_t tiles, char** mem, InstanceLists& lists, cudaStream_t s) {
    static std::once_flag once;
    std::call_once(once, [] {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            unsigned long long keep = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
    });
    const ListLayout ll(R, tiles);
    const cudaError_t e = cudaMallocAsync((void**)mem, ll.bytes, s);
    if (e == cudaSuccess)
        lists = {reinterpret_cast<float*>(*mem + ll.w), reinterpret_cast<uint2*>(*mem + ll.meta),
                 reinterpret_cast<uint32_t*>(*mem + ll.cnt)};
    return e;
}

// The geometry kernel in mode MODE over the view's forward buffers; for EMIT and LIFT also the instance lists and then
// feature_bwd over them (SCORE has neither), reducing sum_p w * scale * map[:, p] into dst.  `a` brings the mode's outputs.  With features
// (EMIT only), feature_dot then turns the lists' weights into pair dot products and the FEAT walk adds the feature term
// to the geometric gradients; the lists are freed after it.
template <BwdMode MODE, typename TG, bool PLANES = false>
static cudaError_t run_bwd(BwdArgs a, const ViewParams& vp, const ForwardBuffers& fb, const TG* map, float scale,
                           float* dst, cudaStream_t s, const FeatureRows& feat = {}) {
    a.pa = producer_args(vp, fb.ranges, fb.point_list, fb.rec, fb.n_contrib, fb.counters + kCounterBwdGeom);
    a.final_T = fb.final_T; a.n_contrib = fb.n_contrib;
    constexpr bool lists = MODE == BwdMode::EMIT || MODE == BwdMode::LIFT;
    char* mem = nullptr;
    if (lists) {
        const cudaError_t e = alloc_lists((size_t)fb.R, (size_t)a.pa.num_tiles, &mem, a.lists, s);
        if (e != cudaSuccess) return e;
    }
    // every instantiation is opted in to the shared memory it needs on the first launch of any of them on a device
    int num_sms = 0;
    cudaError_t e = device_sms<composite_bwd_kernel<BwdMode::GEOM>, composite_bwd_kernel<BwdMode::EMIT>,
                               composite_bwd_kernel<BwdMode::LIFT>, composite_bwd_kernel<BwdMode::FEAT>,
                               composite_bwd_kernel<BwdMode::GEOM, true>, composite_bwd_kernel<BwdMode::EMIT, true>,
                               composite_bwd_kernel<BwdMode::SCORE>>(
        num_sms, sizeof(BwdSmem), kBwdThreads, kSlimCtas);
    const int grid = min(a.pa.num_tiles, kSlimCtas * num_sms);
    auto walk = [&](void (*kernel)(BwdArgs)) {
        cudaError_t ew = cudaMemsetAsync(a.pa.work_counter, 0, sizeof(int), s);
        if (ew != cudaSuccess) return ew;
        kernel<<<grid, kBwdThreads, sizeof(BwdSmem), s>>>(a);
        g_launches++;
        return cudaGetLastError();
    };
    if (e == cudaSuccess) e = walk(composite_bwd_kernel<MODE, PLANES>);
    if (lists) {
        if (e == cudaSuccess) e = launch_feature_bwd(vp, fb.ranges, a.lists, map, scale, dst, fb.counters, s);
        if (MODE == BwdMode::EMIT && feat.rows) {
            if (e == cudaSuccess) e = launch_feature_dot(vp, fb.ranges, a.lists, feat, map, scale, fb.counters, s);
            if (e == cudaSuccess) e = walk(composite_bwd_kernel<BwdMode::FEAT>);
        }
        cudaFreeAsync(mem, s);
    }
    return e;
}

template <typename TG>
cudaError_t launch_composite_bwd(const ViewParams& vp, const ForwardBuffers& fb, const float* bg, const float* dL_dpix,
                                 const float* dL_ddepth, const TG* dL_dfeat_pix, float dL_dfeat_pix_scale,
                                 float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dz,
                                 float* dL_dfeature, cudaStream_t s, const FeatureRows& feat, const float* dL_dalpha,
                                 const float* dL_dinvdepth) {
    BwdArgs a{};
    a.bg = bg; a.dL_dpix = dL_dpix; a.dL_ddepth = dL_ddepth;
    a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic; a.dL_dopacity = dL_dopacity; a.dL_dcolor = dL_dcolor;
    a.dL_dz = dL_dz;
    a.dL_dalpha = dL_dalpha; a.dL_dinvdepth = dL_dinvdepth;
    const bool emit = vp.C > 0 && fb.R > 0;
    const auto run = dL_dalpha ? (emit ? run_bwd<BwdMode::EMIT, TG, true> : run_bwd<BwdMode::GEOM, TG, true>)
                               : (emit ? run_bwd<BwdMode::EMIT, TG> : run_bwd<BwdMode::GEOM, TG>);
    return run(a, vp, fb, dL_dfeat_pix, dL_dfeat_pix_scale, dL_dfeature, s, feat);
}

template <typename TF>
cudaError_t launch_feature_lift(const ViewParams& vp, const ForwardBuffers& fb, const TF* map, float* feature_sum,
                                float* weight_sum, cudaStream_t s) {
    BwdArgs a{};
    a.weight_sum = weight_sum;
    return run_bwd<BwdMode::LIFT>(a, vp, fb, map, 1.f, feature_sum, s);
}

cudaError_t launch_gaussian_scores(const ViewParams& vp, const ForwardBuffers& fb, float* weight_sum, float* max_weight,
                                   int64_t* pixel_count, cudaStream_t s) {
    BwdArgs a{};
    a.weight_sum = weight_sum; a.max_weight = max_weight; a.pixel_count = pixel_count;
    return run_bwd<BwdMode::SCORE, float>(a, vp, fb, nullptr, 1.f, nullptr, s);
}

template cudaError_t launch_composite_bwd(const ViewParams&, const ForwardBuffers&, const float*, const float*,
                                          const float*, const float*, float, float*, float*, float*, float*, float*,
                                          float*, cudaStream_t, const FeatureRows&, const float*, const float*);
template cudaError_t launch_composite_bwd(const ViewParams&, const ForwardBuffers&, const float*, const float*,
                                          const float*, const __half*, float, float*, float*, float*, float*, float*,
                                          float*, cudaStream_t, const FeatureRows&, const float*, const float*);
template cudaError_t launch_feature_lift(const ViewParams&, const ForwardBuffers&, const float*, float*, float*,
                                         cudaStream_t);
template cudaError_t launch_feature_lift(const ViewParams&, const ForwardBuffers&, const __half*, float*, float*,
                                         cudaStream_t);

}  // namespace f3dgs

#ifdef F3DGS_ROLE_CLOCKS
ROLE_CLK_EXPORT(f3dgs_role_clocks_bwd)
#endif
