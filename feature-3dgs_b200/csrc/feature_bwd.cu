// Feature gradient of the two-kernel backward.
//
// The geometric-gradient kernel (composite_bwd.cu, alpha-only layout at two CTAs per SM) appends, per (tile, 8x4 block), one
// list entry per instance that blended at least one pixel of the block: {Gaussian id, pixel mask} + the 32 blend weights
// w = alpha * T (136 bytes per entry, ~6.0 M entries = 0.8 GB per view at config 3, back to front).  Lists need no counting
// pass: block b of tile t owns entries [8*range.x + b*len, ... + len), len = range.y - range.x (an instance of the tile
// list appears at most once per block).
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
#include <cstdio>
#include <cstdlib>

#include "composite_common.cuh"

namespace f3dgs {

constexpr int kListChunk = 16;  // list entries staged per pipeline step (<= 32)
constexpr int kFeatWarps = 4;   // independent worker warps per CTA

struct alignas(128) FeatSmem {  // per warp
    float w[2][kListChunk][32];
};

struct FeatArgs {
    const uint2* ranges;
    const float* list_w;
    const uint2* list_meta;
    const uint32_t* list_cnt;
    const float* dL_dfeat_pix;  // backward: [C, H, W]
    float* dL_dfeature;         // backward: [P, C]
    int* work_counter;
    int W, H, C, tiles_x, num_tiles, chunks;
    int vec;  // bit0: gradient rows are 16-byte aligned and C % 4 == 0; bit1: 4-pixel vector loads of image rows
    // a float16 upstream gradient instead of dL_dfeat_pix: dL/dO = scale * float(map), one fp32 multiply rounded to nearest
    const __half* dL_dfeat_pix_h;
    float scale;
};

__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Decode a work item.  Blocks of one tile are neighbours in the item order, so the workers that run at the same time
// mostly share their instances' feature rows in L2.
struct ItemPos {
    int tile, chunk, b, bx0, by0;
};
__device__ __forceinline__ ItemPos decode_item(int item, const FeatArgs& a) {
    ItemPos p;
    p.b = item & (kBlocksPerTile - 1);
    const int tc = item / kBlocksPerTile;
    p.chunk = tc % a.chunks;
    p.tile = tc / a.chunks;
    const int tile_x = p.tile % a.tiles_x, tile_y = p.tile / a.tiles_x;
    p.bx0 = tile_x * 16 + (p.b & 1) * 8;
    p.by0 = tile_y * 16 + (p.b >> 1) * 4;
    return p;
}

// Loads of the upstream gradient: 4 consecutive pixels (16 bytes of float / 8 bytes of __half, aligned) or one.  A __half
// element is upcast exactly and multiplied by the map's float32 scale once, rounded to nearest.
__device__ __forceinline__ float4 ld_dO4(const float* p, float) { return ld_nc_f4(p); }
__device__ __forceinline__ float4 ld_dO4(const __half* p, float s) {
    uint32_t u0, u1;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(u0), "=r"(u1) : "l"(p));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u0));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u1));
    return make_float4(__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(b.x, s), __fmul_rn(b.y, s));
}
__device__ __forceinline__ float ld_dO1(const float* p, float) { return __ldg(p); }
__device__ __forceinline__ float ld_dO1(const __half* p, float s) { return __fmul_rn(__half2float(__ldg(p)), s); }

// ------------------------------------------------------------------------------------------------ backward
template <int CH, typename TG>  // TG: element type of the upstream gradient map, float or __half
__global__ void __launch_bounds__(kFeatWarps * 32, 3) feature_bwd_kernel(const FeatArgs a) {
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
        const size_t base = 8 * (size_t)rx + (size_t)ip.b * (ry - rx);
        const uint32_t n = __shfl_sync(0xffffffffu, a.list_cnt[(size_t)ip.tile * kBlocksPerTile + ip.b], 0);
        if (n == 0) continue;
        const int ch0 = ip.chunk * CH + cl * 4;
        const uint32_t nch = (n + kListChunk - 1) / kListChunk;

        auto load_meta = [&](uint32_t c) -> uint2 {
            const uint32_t e = c * kListChunk + lane;
            return (lane < kListChunk && e < n) ? __ldg(&a.list_meta[base + e]) : make_uint2(0u, 0u);
        };
        auto issue = [&](uint32_t c, int buf) {
            const uint32_t cnt = min((uint32_t)kListChunk, n - c * kListChunk);
            const float* wsrc = a.list_w + (base + (size_t)c * kListChunk) * 32;
            for (uint32_t j = lane; j < cnt * 8; j += 32) cp_async16(&sm.w[buf][0][0] + j * 4, wsrc + j * 4);
            cp_async_commit();
        };
        uint2 m_cur = load_meta(0);
        issue(0, 0);

        // upstream gradient of the block's 32 pixels x 4 channels: [quad][pixel pair][channel]: the two pixels of a
        // quad row share a 64-bit register pair, as do their weights in the LDS.128
        float2 dO2[NQ][2][4];
#define DOB(q, i, c) (((i) & 1) ? dO2[q][(i) >> 1][c].y : dO2[q][(i) >> 1][c].x)
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
            const TG* plane;
            if constexpr (std::is_same_v<TG, float>)
                plane = a.dL_dfeat_pix + (size_t)ch * HW;
            else
                plane = a.dL_dfeat_pix_h + (size_t)ch * HW;
            if (G == 1 && (a.vec & 2)) {
#pragma unroll
                for (int y = 0; y < 4; y++) {
                    const int yy = ip.by0 + y;
                    if (yy >= H) continue;
#pragma unroll
                    for (int half = 0; half < 2; half++) {
                        const int xx = ip.bx0 + half * 4;
                        if (xx >= W) continue;
                        const int qa = (y >> 1) * 4 + half * 2, i0 = (y & 1) * 2;
                        const float4 v = ld_dO4(plane + (size_t)yy * W + xx, a.scale);
                        DOB(qa % NQ, i0, c) = v.x;
                        DOB(qa % NQ, i0 + 1, c) = v.y;
                        DOB((qa + 1) % NQ, i0, c) = v.z;
                        DOB((qa + 1) % NQ, i0 + 1, c) = v.w;
                    }
                }
            } else {
#pragma unroll
                for (int qi = 0; qi < NQ; qi++) {
                    const int q = qi * G + grp;
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const int xx = ip.bx0 + (q & 3) * 2 + (i & 1), yy = ip.by0 + (q >> 2) * 2 + (i >> 1);
                        if (xx < W && yy < H) DOB(qi, i, c) = ld_dO1(plane + (size_t)yy * W + xx, a.scale);
                    }
                }
            }
        }
#undef DOB

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

// ------------------------------------------------------------------------------------------------ launchers
static int workers_grid() {
    static std::atomic<int> sms_of_device[64];  // zero-initialised; set once per device (idempotent)
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return 132 * 3;
    if (sms_of_device[dev].load() == 0) {
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sms_of_device[dev].store(n > 0 ? n : 132);
    }
    return sms_of_device[dev].load() * 3;  // __launch_bounds__(128, 3): three CTAs of four workers per SM
}

template <int CH, typename TG>
static cudaError_t launch_feat_bwd_t(const FeatArgs& a, cudaStream_t s) {
    const size_t smem = kFeatWarps * sizeof(FeatSmem);
    const int items = a.num_tiles * a.chunks * kBlocksPerTile;
    const int grid = min((items + kFeatWarps - 1) / kFeatWarps, workers_grid());
    feature_bwd_kernel<CH, TG><<<grid, kFeatWarps * 32, smem, s>>>(a);
    g_launches++;
    return cudaGetLastError();
}

static int feat_ch(int C) { return C <= 32 ? 32 : (C <= 64 ? 64 : 128); }

template <typename TG>
cudaError_t launch_feature_bwd(const ViewParams& vp, const uint2* ranges, const float* list_w, const uint2* list_meta,
                               const uint32_t* list_cnt, const TG* dL_dfeat_pix, float dL_dfeat_pix_scale,
                               float* dL_dfeature, int* work_counter, cudaStream_t s) {
    FeatArgs a;
    a.ranges = ranges; a.list_w = list_w; a.list_meta = list_meta; a.list_cnt = list_cnt;
    if constexpr (std::is_same_v<TG, float>) {
        a.dL_dfeat_pix = dL_dfeat_pix; a.dL_dfeat_pix_h = nullptr;
    } else {
        a.dL_dfeat_pix = nullptr; a.dL_dfeat_pix_h = dL_dfeat_pix;
    }
    a.dL_dfeature = dL_dfeature; a.scale = dL_dfeat_pix_scale;
    a.work_counter = work_counter;
    a.W = vp.W; a.H = vp.H; a.C = vp.C; a.tiles_x = (int)vp.grid_x; a.num_tiles = (int)(vp.grid_x * vp.grid_y);
    const int CH = feat_ch(vp.C);
    a.chunks = (vp.C + CH - 1) / CH;
    a.vec = 0;
    if (vp.C % 4 == 0 && (reinterpret_cast<uintptr_t>(dL_dfeature) & 15) == 0) a.vec |= 1;
    if (vp.W % 4 == 0 && (reinterpret_cast<uintptr_t>(dL_dfeat_pix) & (4 * sizeof(TG) - 1)) == 0) a.vec |= 2;
    cudaError_t e = cudaMemsetAsync(work_counter, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    if (CH == 32) return launch_feat_bwd_t<32, TG>(a, s);
    if (CH == 64) return launch_feat_bwd_t<64, TG>(a, s);
    return launch_feat_bwd_t<128, TG>(a, s);
}
template cudaError_t launch_feature_bwd(const ViewParams&, const uint2*, const float*, const uint2*, const uint32_t*,
                                       const float*, float, float*, int*, cudaStream_t);
template cudaError_t launch_feature_bwd(const ViewParams&, const uint2*, const float*, const uint2*, const uint32_t*,
                                       const __half*, float, float*, int*, cudaStream_t);

}  // namespace f3dgs
