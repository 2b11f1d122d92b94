// Tile binning: (tile | depth) key emission and per-tile range detection.
//
//   duplicate_keys_kernel : reference duplicateWithKeys, rasterizer_impl.cu:70-111
//   tile_ranges_kernel    : reference identifyTileRanges, rasterizer_impl.cu:116-138
//
// Bit-exact contract: key = (tile_id << 32) | float_bits(depth), emitted y-outer / x-inner inside
// the Gaussian's rectangle starting at offsets[i-1]; the sort (cub::DeviceRadixSort, api.cu) is
// stable, so equal keys keep ascending Gaussian order.
//
// Notes: emission is warp-cooperative -- a warp owns 32 consecutive Gaussians and spreads
// the (Gaussian, tile) instances of all of them over its lanes, so one huge splat does not
// serialise a thread (the reference loops per thread) and the 12-byte-per-instance stores are
// coalesced runs.
#include "kernels.h"

namespace f3dgs {

__global__ void __launch_bounds__(256)
duplicate_keys_kernel(int P, const SplatRec* __restrict__ rec, const uint32_t* __restrict__ offsets,
                      const int* __restrict__ radii, uint32_t grid_x, uint32_t grid_y,
                      uint64_t* __restrict__ keys, uint32_t* __restrict__ values) {
    const int lane = threadIdx.x & 31;
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int base = warp_global * 32;
    if (base >= P) return;
    const int idx = base + lane;

    uint32_t x0 = 0, y0 = 0, w = 0, n = 0, off = 0, depth_bits = 0;
    if (idx < P) {
        const int r = radii[idx];
        if (r > 0) {
            const float4 g0 = reinterpret_cast<const float4*>(rec + idx)[0];
            depth_bits = __float_as_uint(reinterpret_cast<const float4*>(rec + idx)[2].w);
            uint32_t x1, y1;
            tile_rect(g0.x, g0.y, r, grid_x, grid_y, x0, y0, x1, y1);
            w = x1 - x0;
            n = w * (y1 - y0);
            off = (idx == 0) ? 0u : offsets[idx - 1];
        }
    }
    // Small rectangles: the owning lane writes them itself.  Large ones are spread over the warp.
    constexpr uint32_t kCoop = 32;
    if (n > 0 && n < kCoop) {
        uint32_t o = off;
        for (uint32_t yy = 0, cnt = 0; cnt < n; yy++)
            for (uint32_t xx = 0; xx < w; xx++, cnt++) {
                const uint64_t key = ((uint64_t)((y0 + yy) * grid_x + (x0 + xx)) << 32) | depth_bits;
                keys[o] = key;
                values[o] = (uint32_t)idx;
                o++;
            }
    }
    uint32_t big = __ballot_sync(0xffffffffu, n >= kCoop);
    while (big) {
        const int src = __ffs(big) - 1;
        big &= big - 1;
        const uint32_t bx0 = __shfl_sync(0xffffffffu, x0, src);
        const uint32_t by0 = __shfl_sync(0xffffffffu, y0, src);
        const uint32_t bw = __shfl_sync(0xffffffffu, w, src);
        const uint32_t bn = __shfl_sync(0xffffffffu, n, src);
        const uint32_t boff = __shfl_sync(0xffffffffu, off, src);
        const uint32_t bd = __shfl_sync(0xffffffffu, depth_bits, src);
        for (uint32_t i = lane; i < bn; i += 32) {
            const uint32_t yy = i / bw, xx = i - yy * bw;
            keys[boff + i] = ((uint64_t)((by0 + yy) * grid_x + (bx0 + xx)) << 32) | bd;
            values[boff + i] = (uint32_t)(base + src);
        }
    }
}

__global__ void __launch_bounds__(256)
tile_ranges_kernel(int R, const uint64_t* __restrict__ sorted_keys, uint2* __restrict__ ranges) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= R) return;
    const uint32_t cur = (uint32_t)(sorted_keys[idx] >> 32);
    if (idx == 0) {
        ranges[cur].x = 0;
    } else {
        const uint32_t prev = (uint32_t)(sorted_keys[idx - 1] >> 32);
        if (cur != prev) {
            ranges[prev].y = idx;
            ranges[cur].x = idx;
        }
    }
    if (idx == R - 1) ranges[cur].y = R;
}

void launch_duplicate_keys(int P, const SplatRec* rec, const uint32_t* offsets, const int* radii,
                           uint32_t grid_x, uint32_t grid_y, uint64_t* keys, uint32_t* values,
                           cudaStream_t s) {
    if (P <= 0) return;
    duplicate_keys_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, rec, offsets, radii, grid_x, grid_y, keys, values);
    g_launches++;
}

void launch_tile_ranges(int R, const uint64_t* sorted_keys, uint2* ranges, cudaStream_t s) {
    if (R <= 0) return;
    tile_ranges_kernel<<<(R + 255) / 256, 256, 0, s>>>(R, sorted_keys, ranges);
    g_launches++;
}

}  // namespace f3dgs
