// Feature gradient of the two-kernel backward.
//
// The geometric-gradient kernel (composite_bwd.cu, alpha-only layout at two CTAs per SM) appends, per (tile, 8x4 block), one
// list entry per instance that blended at least one pixel of the block: {Gaussian id, pixel mask} + the 32 blend weights
// w = alpha * T (136 bytes per entry, ~6.0 M entries = 0.8 GB per view at config 3, back to front), laid out by list_begin.
//
// feature_bwd_kernel<CH> (here): every warp is an independent worker that pulls (tile, channel chunk, block) items from an
// atomic counter, keeps the block's upstream gradient dL/dfeature_map (32 pixels x 4 channels per lane) in registers,
// streams the block's list through a double-buffered cp.async ring (16 entries per step) and forms
// dL/df[g] += sum_pixels w * dL/dO with paired FMAs (fma2_rn) over the 2x2-pixel quads that blended, one red.global.add.v4
// per lane and entry.  No inter-warp synchronisation at all; 12 warps per SM.  Channel counts above 128 reuse the same
// lists for every 128-channel chunk (the alpha evaluation is not repeated per chunk).
// The upstream gradient may be a float16 map h with a float32 scale s (training float16 feature fields): it is upcast and
// multiplied by s once, where the block's gradient is loaded, and everything after that is the float32 kernel.
// Reference semantics: backward.cu:565-575 (feature gradient; the feature loss does not feed dL/dalpha, :575 disabled).
//
// feature_dot_kernel<CH> (here, opt-in): the pair dot products d_ip = f_i . dL/dfeature_map[:, p] for the feature term
// of dL/dalpha (composite_bwd.cu, FEAT).  One warp per (tile, block) item walks the block's list once per CH-channel
// chunk, with the block's gradient chunk in registers exactly as above, gathers each entry's feature-row chunk (4
// channels per lane) and forms its partial dot product at each of the lane's pixels; a reduce-scatter over the CH / 4
// lanes that share those pixels leaves each lane with the chunk's whole dot product at one pixel.  The first chunk
// stores it into the entry's weight row, which feature_bwd is done with, and later chunks add to it: the warp owns the
// rows of its item, so there are no atomics and the result is deterministic.
#include <cstdio>
#include <cstdlib>

#include "composite_common.cuh"

namespace f3dgs {

constexpr int kListChunk = 16;  // list entries staged per pipeline step (<= 32)
constexpr int kFeatWarps = 4;   // independent worker warps per CTA

struct alignas(128) FeatSmem {  // per warp
    float w[2][kListChunk][32];
};

template <typename TG>  // TG: element type of the upstream gradient map, float or __half
struct FeatArgs {
    const uint2* ranges;
    InstanceLists lists;
    const TG* dL_dfeat_pix;  // backward: [C, H, W]
    float* dL_dfeature;      // backward: [P, C]
    int* work_counter;
    int W, H, C, tiles_x, num_tiles, chunks;
    int vec;  // bit0: gradient rows are 16-byte aligned and C % 4 == 0; bit1: 4-pixel vector loads of image rows
    // a float16 map stands for dL/dO = scale * float(map), one fp32 multiply rounded to nearest; not read for float
    float scale;
};

// Decode a work item.  Blocks of one tile are neighbours in the item order, so the workers that run at the same time
// mostly share their instances' feature rows in L2.
struct ItemPos {
    int tile, chunk, b, bx0, by0;
};
template <typename TG>
__device__ __forceinline__ ItemPos decode_item(int item, const FeatArgs<TG>& a) {
    ItemPos p;
    p.b = item & (kBlocksPerTile - 1);
    const int tc = item / kBlocksPerTile;
    p.chunk = tc % a.chunks;
    p.tile = tc / a.chunks;
    const int tile_x = p.tile % a.tiles_x, tile_y = p.tile / a.tiles_x;
    p.bx0 = block_x0(tile_x, p.b);
    p.by0 = block_y0(tile_y, p.b);
    return p;
}

// Loads of the upstream gradient: 4 consecutive pixels (16 bytes of float / 8 bytes of __half, aligned) or one.  A __half
// element is upcast exactly and multiplied by the map's float32 scale once, rounded to nearest.
__device__ __forceinline__ float4 ld_dO4(const float* p, float) { return ld_nc_f4(p); }
__device__ __forceinline__ float4 ld_dO4(const __half* p, float s) {
    uint32_t u0, u1;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(u0), "=r"(u1) : "l"(p));
    const float4 v = to_float4(make_uint2(u0, u1));
    return make_float4(__fmul_rn(v.x, s), __fmul_rn(v.y, s), __fmul_rn(v.z, s), __fmul_rn(v.w, s));
}
__device__ __forceinline__ float ld_dO1(const float* p, float) { return __ldg(p); }
__device__ __forceinline__ float ld_dO1(const __half* p, float s) { return __fmul_rn(__half2float(__ldg(p)), s); }

// ------------------------------------------------------------------------------------------------ backward
template <int CH, typename TG>
__global__ void __launch_bounds__(kFeatWarps * 32, 3) feature_bwd_kernel(const FeatArgs<TG> a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    FeatSmem& sm = reinterpret_cast<FeatSmem*>(smem_raw)[warp];
    constexpr int LPR = CH / 4;
    constexpr int G = 32 / LPR;
    constexpr int NQ = 8 / G;
    const int grp = lane / LPR, cl = lane % LPR;
    const int W = a.W, H = a.H, C = a.C;
    const size_t HW = (size_t)H * W;

    const int items = a.num_tiles * a.chunks * kBlocksPerTile;
    for (;;) {
        int item = 0;
        if (lane == 0) item = atomicAdd(a.work_counter, 1);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= items) break;
        const ItemPos ip = decode_item(item, a);
        // loaded from uniform addresses, but only a shuffle tells ptxas that the values are warp-uniform (uniform loop
        // trip counts and branches: no reconvergence pairs around the quad tests)
        const uint32_t rx = __shfl_sync(0xffffffffu, a.ranges[ip.tile].x, 0);
        const uint32_t ry = __shfl_sync(0xffffffffu, a.ranges[ip.tile].y, 0);
        const size_t base = list_begin(rx, ry, ip.b);
        const uint32_t n = __shfl_sync(0xffffffffu, a.lists.cnt[(size_t)ip.tile * kBlocksPerTile + ip.b], 0);
        if (n == 0) continue;
        const int ch0 = ip.chunk * CH + cl * 4;
        const uint32_t nch = (n + kListChunk - 1) / kListChunk;

        auto load_meta = [&](uint32_t c) -> uint2 {
            const uint32_t e = c * kListChunk + lane;
            return (lane < kListChunk && e < n) ? __ldg(&a.lists.meta[base + e]) : make_uint2(0u, 0u);
        };
        auto issue = [&](uint32_t c, int buf) {
            const uint32_t cnt = min((uint32_t)kListChunk, n - c * kListChunk);
            const float* wsrc = a.lists.w + (base + (size_t)c * kListChunk) * 32;
            for (uint32_t j = lane; j < cnt * 8; j += 32) cp_async16(&sm.w[buf][0][0] + j * 4, wsrc + j * 4);
            cp_async_commit();
        };
        uint2 m_cur = load_meta(0);
        issue(0, 0);

        // upstream gradient of the block's 32 pixels x 4 channels: [quad][pixel pair][channel]: the two pixels of a
        // quad row share a 64-bit register pair, as do their weights in the LDS.128
        float2 dO2[NQ][2][4];
#pragma unroll
        for (int q = 0; q < NQ; q++)
#pragma unroll
            for (int r = 0; r < 2; r++)
#pragma unroll
                for (int c = 0; c < 4; c++) dO2[q][r][c] = make_float2(0.f, 0.f);
#pragma unroll
        for (int c = 0; c < 4; c++) {
            const int ch = ch0 + c;
            if (ch >= C) continue;
            for_tile_pixels<G, NQ>(
                a.dL_dfeat_pix + (size_t)ch * HW, ip.bx0, ip.by0, W, H, grp, false, a.vec & 2, [](const TG*, int) {},
                [&](const TG* p, int y, int half) { set_tile_run(dO2, y, half, c, ld_dO4(p, a.scale)); },
                [&](const TG* p, int qi, int i) { tile_px(dO2, qi, i, c) = ld_dO1(p, a.scale); });
        }

        for (uint32_t c = 0; c < nch; c++) {
            const int buf = c & 1;
            const uint2 m_nxt = load_meta(c + 1);
            if (c + 1 < nch) {
                issue(c + 1, buf ^ 1);
                cp_async_wait<1>();
            } else {
                cp_async_wait<0>();
            }
            __syncwarp();
            const uint32_t cnt = min((uint32_t)kListChunk, n - c * kListChunk);
            for (uint32_t i = 0; i < cnt; i++) {
                const uint32_t gid = __shfl_sync(0xffffffffu, m_cur.x, i);
                const uint32_t pm = __shfl_sync(0xffffffffu, m_cur.y, i);
                float2 gp[4];  // per channel: (sum over even pixel columns, sum over odd pixel columns)
#pragma unroll
                for (int ch = 0; ch < 4; ch++) gp[ch] = make_float2(0.f, 0.f);
#pragma unroll
                for (int qi = 0; qi < NQ; qi++) {
                    const int q = qi * G + grp;
                    if ((pm >> (4 * q)) & 0xFu) {
                        const float4 w4 = *reinterpret_cast<const float4*>(&sm.w[buf][i][4 * q]);
                        const float2 w01 = make_float2(w4.x, w4.y), w23 = make_float2(w4.z, w4.w);
#pragma unroll
                        for (int ch = 0; ch < 4; ch++) gp[ch] = fma2_rn(w01, dO2[qi][0][ch], gp[ch]);
#pragma unroll
                        for (int ch = 0; ch < 4; ch++) gp[ch] = fma2_rn(w23, dO2[qi][1][ch], gp[ch]);
                    }
                }
                float g0 = gp[0].x + gp[0].y, g1 = gp[1].x + gp[1].y, g2 = gp[2].x + gp[2].y, g3 = gp[3].x + gp[3].y;
#pragma unroll
                for (int o = LPR; o < 32; o <<= 1) {
                    g0 += __shfl_xor_sync(0xffffffffu, g0, o);
                    g1 += __shfl_xor_sync(0xffffffffu, g1, o);
                    g2 += __shfl_xor_sync(0xffffffffu, g2, o);
                    g3 += __shfl_xor_sync(0xffffffffu, g3, o);
                }
                if (grp == 0 && ch0 < C) {
                    float* dst = a.dL_dfeature + (size_t)gid * C + ch0;
                    if (a.vec & 1) {
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
            m_cur = m_nxt;
        }
    }
}

// ------------------------------------------------------------------------------------------------ pair dot products
template <typename TF, typename TG>
struct DotArgs {
    FeatArgs<TG> f;      // bit0 of f.vec: feature rows are 4-channel aligned (C % 4 == 0 and an aligned base)
    const TF* features;  // [P, C]
};

// Four channels of a feature row, a float16 row upcast exactly as the forward reads it
__device__ __forceinline__ float4 ld_feat4(const float* p) { return ld_nc_f4(p); }
__device__ __forceinline__ float4 ld_feat4(const __half* p) {
    uint32_t u0, u1;
    asm volatile("ld.global.nc.v2.u32 {%0,%1}, [%2];" : "=r"(u0), "=r"(u1) : "l"(p));
    return to_float4(make_uint2(u0, u1));
}
__device__ __forceinline__ float ld_feat1(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld_feat1(const __half* p) { return __half2float(__ldg(p)); }

// c ? x : y as one SELP: spelled as a select, the compiler turns the reduce-scatter's selects into a dynamically indexed
// array in local memory
__device__ __forceinline__ float sel(uint32_t c, float x, float y) {
    float r;
    asm("{.reg .pred p; setp.ne.u32 p, %3, 0; selp.f32 %0, %1, %2, p;}" : "=f"(r) : "f"(x), "f"(y), "r"(c));
    return r;
}

template <int CH, typename TF, typename TG>
__global__ void __launch_bounds__(kFeatWarps * 32, 3) feature_dot_kernel(const DotArgs<TF, TG> d) {
    const FeatArgs<TG>& a = d.f;
    const int lane = threadIdx.x & 31;
    constexpr int LPR = CH / 4;  // lanes per feature row = pixels per lane
    constexpr int G = 32 / LPR;
    constexpr int NQ = 8 / G;
    const int grp = lane / LPR, cl = lane % LPR;
    // after the reduce-scatter lane (grp, cl) holds the lane group's pixel cl: pixel cl & 3 of its quad cl >> 2
    const int slot = 4 * ((cl >> 2) * G + grp) + (cl & 3);
    const int W = a.W, H = a.H, C = a.C;
    const size_t HW = (size_t)H * W;

    const int items = a.num_tiles * kBlocksPerTile;
    for (;;) {
        int item = 0;
        if (lane == 0) item = atomicAdd(a.work_counter, 1);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= items) break;
        const int tile = item / kBlocksPerTile, b = item % kBlocksPerTile;
        const int bx0 = block_x0(tile % a.tiles_x, b), by0 = block_y0(tile / a.tiles_x, b);
        const uint32_t rx = __shfl_sync(0xffffffffu, a.ranges[tile].x, 0);
        const uint32_t ry = __shfl_sync(0xffffffffu, a.ranges[tile].y, 0);
        const size_t base = list_begin(rx, ry, b);
        const uint32_t n = __shfl_sync(0xffffffffu, a.lists.cnt[(size_t)tile * kBlocksPerTile + b], 0);
        if (n == 0) continue;

        for (int chunk = 0; chunk < a.chunks; chunk++) {
            const int ch0 = chunk * CH + cl * 4;
            float2 dO2[NQ][2][4];  // as in feature_bwd_kernel
#pragma unroll
            for (int q = 0; q < NQ; q++)
#pragma unroll
                for (int r = 0; r < 2; r++)
#pragma unroll
                    for (int c = 0; c < 4; c++) dO2[q][r][c] = make_float2(0.f, 0.f);
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int ch = ch0 + c;
                if (ch >= C) continue;
                for_tile_pixels<G, NQ>(
                    a.dL_dfeat_pix + (size_t)ch * HW, bx0, by0, W, H, grp, false, a.vec & 2, [](const TG*, int) {},
                    [&](const TG* p, int y, int half) { set_tile_run(dO2, y, half, c, ld_dO4(p, a.scale)); },
                    [&](const TG* p, int qi, int i) { tile_px(dO2, qi, i, c) = ld_dO1(p, a.scale); });
            }

            for (uint32_t c0 = 0; c0 < n; c0 += 32) {
                const uint2 m = c0 + lane < n ? __ldg(&a.lists.meta[base + c0 + lane]) : make_uint2(0u, 0u);
                const uint32_t cnt = min(32u, n - c0);
                // the entry's feature-row chunk, loaded one entry ahead of its use
                auto load_row = [&](uint32_t gid) {
                    float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
                    const TF* src = d.features + (size_t)gid * C + ch0;
                    if (ch0 < C) {
                        if (a.vec & 1) {
                            f = ld_feat4(src);
                        } else {
                            f.x = ld_feat1(src);
                            if (ch0 + 1 < C) f.y = ld_feat1(src + 1);
                            if (ch0 + 2 < C) f.z = ld_feat1(src + 2);
                            if (ch0 + 3 < C) f.w = ld_feat1(src + 3);
                        }
                    }
                    return f;
                };
                float4 f_nxt = load_row(__shfl_sync(0xffffffffu, m.x, 0));
#pragma unroll 1
                for (uint32_t i = 0; i < cnt; i++) {
                    const uint32_t pm = __shfl_sync(0xffffffffu, m.y, i);
                    const float4 f = f_nxt;
                    const uint32_t gid_nxt = __shfl_sync(0xffffffffu, m.x, (i + 1) & 31);
                    if (i + 1 < cnt) f_nxt = load_row(gid_nxt);
                    // partial dot product at each of the lane's pixels, pixel i of its quad qi at index 4 qi + i (0 where
                    // the quad did not blend: the FEAT walk reads only the blended pixels), then a reduce-scatter over the
                    // LPR lanes of the group: at offset o the lane keeps the half of its values selected by bit o of cl and
                    // adds its partner's copy of that half.  The first step (o = LPR / 2: quads qi and qi + NQ / 2) is
                    // taken as the values are formed, so that only half of them are ever live.
                    auto dot = [&](int qi, int r) {
                        float2 acc = make_float2(0.f, 0.f);
                        if ((pm >> (4 * (qi * G + grp))) & 0xFu) {
                            acc = fma2_rn(make_float2(f.x, f.x), dO2[qi][r][0], acc);
                            acc = fma2_rn(make_float2(f.y, f.y), dO2[qi][r][1], acc);
                            acc = fma2_rn(make_float2(f.z, f.z), dO2[qi][r][2], acc);
                            acc = fma2_rn(make_float2(f.w, f.w), dO2[qi][r][3], acc);
                        }
                        return acc;
                    };
                    constexpr int H2 = LPR / 2;
                    float v[H2];
                    {
                        const uint32_t up = cl & H2;
#pragma unroll
                        for (int qi = 0; qi < NQ / 2; qi++)
#pragma unroll
                            for (int r = 0; r < 2; r++) {
                                const float2 lo = dot(qi, r), hi = dot(qi + NQ / 2, r);
                                v[4 * qi + 2 * r] = sel(up, hi.x, lo.x) + __shfl_xor_sync(0xffffffffu, sel(up, lo.x, hi.x), H2);
                                v[4 * qi + 2 * r + 1] =
                                    sel(up, hi.y, lo.y) + __shfl_xor_sync(0xffffffffu, sel(up, lo.y, hi.y), H2);
                            }
                    }
#pragma unroll
                    for (int o = H2 / 2; o > 0; o >>= 1) {
                        const uint32_t up = cl & o;
#pragma unroll
                        for (int j = 0; j < o; j++) {
                            const float send = sel(up, v[j], v[j + o]);
                            const float keep = sel(up, v[j + o], v[j]);
                            v[j] = keep + __shfl_xor_sync(0xffffffffu, send, o);
                        }
                    }
                    float* dst = a.lists.w + (base + c0 + i) * 32 + slot;
                    *dst = chunk == 0 ? v[0] : *dst + v[0];
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ launchers
template <int CH, typename TG>
static cudaError_t launch_feat_bwd_t(const FeatArgs<TG>& a, cudaStream_t s) {
    const size_t smem = kFeatWarps * sizeof(FeatSmem);  // under 48 KB: no opt-in
    int sms = 132;  // kept for a device ordinal device_sms does not cover
    device_sms<>(sms, smem);
    const int items = a.num_tiles * a.chunks * kBlocksPerTile;
    // __launch_bounds__(128, 3): three CTAs of four workers per SM
    const int grid = min((items + kFeatWarps - 1) / kFeatWarps, sms * 3);
    feature_bwd_kernel<CH, TG><<<grid, kFeatWarps * 32, smem, s>>>(a);
    g_launches++;
    return cudaGetLastError();
}

template <typename TG>
cudaError_t launch_feature_bwd(const ViewParams& vp, const uint2* ranges, const InstanceLists& lists,
                               const TG* dL_dfeat_pix, float dL_dfeat_pix_scale, float* dL_dfeature, int* counters,
                               cudaStream_t s) {
    FeatArgs<TG> a;
    a.ranges = ranges; a.lists = lists;
    a.dL_dfeat_pix = dL_dfeat_pix;
    a.dL_dfeature = dL_dfeature; a.scale = dL_dfeat_pix_scale;
    a.work_counter = counters + kCounterFeatureBwd;
    a.W = vp.W; a.H = vp.H; a.C = vp.C; a.tiles_x = (int)vp.grid_x; a.num_tiles = (int)(vp.grid_x * vp.grid_y);
    const int CH = channel_chunk(vp.C);
    a.chunks = (vp.C + CH - 1) / CH;
    a.vec = 0;
    if (vp.C % 4 == 0 && (reinterpret_cast<uintptr_t>(dL_dfeature) & 15) == 0) a.vec |= 1;
    if (vp.W % 4 == 0 && (reinterpret_cast<uintptr_t>(dL_dfeat_pix) & (4 * sizeof(TG) - 1)) == 0) a.vec |= 2;
    cudaError_t e = cudaMemsetAsync(a.work_counter, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    if (CH == 32) return launch_feat_bwd_t<32, TG>(a, s);
    if (CH == 64) return launch_feat_bwd_t<64, TG>(a, s);
    return launch_feat_bwd_t<128, TG>(a, s);
}
template cudaError_t launch_feature_bwd(const ViewParams&, const uint2*, const InstanceLists&, const float*, float,
                                       float*, int*, cudaStream_t);
template cudaError_t launch_feature_bwd(const ViewParams&, const uint2*, const InstanceLists&, const __half*, float,
                                       float*, int*, cudaStream_t);

template <int CH, typename TF, typename TG>
static cudaError_t launch_feat_dot_t(const DotArgs<TF, TG>& d, cudaStream_t s) {
    int sms = 132;  // kept for a device ordinal device_sms does not cover
    device_sms<>(sms, 0);
    const int items = d.f.num_tiles * kBlocksPerTile;
    const int grid = min((items + kFeatWarps - 1) / kFeatWarps, sms * 3);
    feature_dot_kernel<CH, TF, TG><<<grid, kFeatWarps * 32, 0, s>>>(d);
    g_launches++;
    return cudaGetLastError();
}

template <typename TF, typename TG>
static cudaError_t launch_feat_dot_tf(const DotArgs<TF, TG>& d, cudaStream_t s) {
    const int CH = channel_chunk(d.f.C);
    if (CH == 32) return launch_feat_dot_t<32>(d, s);
    if (CH == 64) return launch_feat_dot_t<64>(d, s);
    return launch_feat_dot_t<128>(d, s);
}

template <typename TG>
cudaError_t launch_feature_dot(const ViewParams& vp, const uint2* ranges, const InstanceLists& lists,
                               const FeatureRows& feat, const TG* dL_dfeat_pix, float dL_dfeat_pix_scale, int* counters,
                               cudaStream_t s) {
    FeatArgs<TG> a;
    a.ranges = ranges; a.lists = lists;
    a.dL_dfeat_pix = dL_dfeat_pix; a.scale = dL_dfeat_pix_scale;
    a.dL_dfeature = nullptr;
    a.work_counter = counters + kCounterFeatureBwd;
    a.W = vp.W; a.H = vp.H; a.C = vp.C; a.tiles_x = (int)vp.grid_x; a.num_tiles = (int)(vp.grid_x * vp.grid_y);
    a.chunks = (vp.C + channel_chunk(vp.C) - 1) / channel_chunk(vp.C);
    a.vec = 0;
    const size_t fsz = feat.f16 ? sizeof(__half) : sizeof(float);
    if (vp.C % 4 == 0 && (reinterpret_cast<uintptr_t>(feat.rows) & (4 * fsz - 1)) == 0) a.vec |= 1;
    if (vp.W % 4 == 0 && (reinterpret_cast<uintptr_t>(dL_dfeat_pix) & (4 * sizeof(TG) - 1)) == 0) a.vec |= 2;
    const cudaError_t e = cudaMemsetAsync(a.work_counter, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    if (feat.f16) return launch_feat_dot_tf(DotArgs<__half, TG>{a, static_cast<const __half*>(feat.rows)}, s);
    return launch_feat_dot_tf(DotArgs<float, TG>{a, static_cast<const float*>(feat.rows)}, s);
}
template cudaError_t launch_feature_dot(const ViewParams&, const uint2*, const InstanceLists&, const FeatureRows&,
                                       const float*, float, int*, cudaStream_t);
template cudaError_t launch_feature_dot(const ViewParams&, const uint2*, const InstanceLists&, const FeatureRows&,
                                       const __half*, float, int*, cudaStream_t);

}  // namespace f3dgs
