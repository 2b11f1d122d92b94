// Post-raster feature head (SURVEY.md section 8 f1): bilinear resize of the rendered feature map to the teacher's
// resolution fused with the L1 feature loss and its gradient.
// Reference: train.py:98-104
//     feature_map = F.interpolate(feature_map.unsqueeze(0), size=gt.shape[1:], mode='bilinear', align_corners=True)
//     [feature_map = cnn_decoder(feature_map)]                       (models/networks.py:107-119, only with --speedup)
//     Ll1_feature = l1_loss(feature_map, gt_feature_map)             (utils/loss_utils.py: mean |a - b|)
// In PyTorch that is a resize kernel (write C*Hg*Wg), an L1 kernel pair, and in the backward a sign kernel, a scatter of
// the resize gradient with atomics into a zero-filled C*H*W tensor.  Here:
//     resize_fwd   reads the C*H*W map once; with a target it writes  sign(interp - gt) * grad_scale  (the gradient of the
//                  loss w.r.t. the resized map, ready for the backward) and accumulates sum |interp - gt|; without a
//                  target it writes the resized map (decoder path: feature_decoder.cu runs the 1x1 convolution and
//                  its loss in between).
//     resize_bwd   GATHERS: one thread per element of the C*H*W gradient sums the (few) target pixels whose bilinear
//                  footprint covers it -- every element written exactly once, no atomics, no zero fill.
// Sampling positions follow ATen's upsample_bilinear2d with align_corners=True: src = dst * (in - 1) / (out - 1),
// i0 = (int)src, i1 = i0 + (i0 < in - 1), lambda1 = src - i0.
// The target may be float32 or float16 (the data format's teacher maps); a float16 element is upcast exactly at its load,
// so the result equals that of the float32 target gt.float().
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>

#include "../../include/f3dgs_b200.h"
#include "kernels.h"
#include "tf32_mma.cuh"

namespace f3dgs {
namespace {

struct ResizeGeom {
    int C, H, W, Hg, Wg;
    float ry, rx;  // (in - 1) / (out - 1), 0 when out == 1
};

__device__ __forceinline__ void src_of(int o, float r, int in, int& i0, int& i1, float& l0, float& l1) {
    const float s = r * (float)o;
    i0 = (int)s;
    i1 = i0 + ((i0 < in - 1) ? 1 : 0);
    l1 = s - (float)i0;
    l0 = 1.0f - l1;
}

// One warp per output row (c, oy) at a time, lanes strided over ox: the row's channel plane and y taps are computed once per
// row (no per-element division), a lane's loads are independent across its elements, and consecutive lanes read source
// columns (in - 1) / (out - 1) apart -- neighbouring sectors.  A persistent grid, so that the loss needs one atomic per CTA
// (200 K same-address atomics cost more than the whole resize).
constexpr int kFwdThreads = 256;

template <typename GT>  // float or __half
__global__ void __launch_bounds__(kFwdThreads) resize_fwd_kernel(ResizeGeom g, const float* __restrict__ fm,
                                                                 const GT* __restrict__ gt, float grad_scale,
                                                                 float* __restrict__ out, float* __restrict__ loss_sum) {
    const int lane = threadIdx.x & 31;
    const int warps = gridDim.x * (kFwdThreads / 32);
    const int rows = g.C * g.Hg;
    float ad = 0.f;
    for (int row = blockIdx.x * (kFwdThreads / 32) + (threadIdx.x >> 5); row < rows; row += warps) {
        const int c = row / g.Hg, oy = row - c * g.Hg;
        int y0, y1;
        float ly0, ly1;
        src_of(oy, g.ry, g.H, y0, y1, ly0, ly1);
        const float* p0 = fm + ((size_t)c * g.H + y0) * g.W;
        const float* p1 = fm + ((size_t)c * g.H + y1) * g.W;
        const size_t obase = (size_t)row * g.Wg;
#pragma unroll 2
        for (int ox = lane; ox < g.Wg; ox += 32) {
            int x0, x1;
            float lx0, lx1;
            src_of(ox, g.rx, g.W, x0, x1, lx0, lx1);
            const float v = ly0 * (lx0 * __ldg(p0 + x0) + lx1 * __ldg(p0 + x1)) + ly1 * (lx0 * __ldg(p1 + x0) + lx1 * __ldg(p1 + x1));
            if (gt != nullptr) {
                const float d = v - load_f32(gt + obase + ox);
                ad += fabsf(d);
                out[obase + ox] = d > 0.f ? grad_scale : (d < 0.f ? -grad_scale : 0.f);
            } else {
                out[obase + ox] = v;
            }
        }
    }
    if (gt != nullptr && loss_sum != nullptr) {
        // block reduction of |d|, one atomic per block
        __shared__ float part[kFwdThreads / 32];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ad += __shfl_xor_sync(0xffffffffu, ad, o);
        if (lane == 0) part[threadIdx.x >> 5] = ad;
        __syncthreads();
        if (threadIdx.x < kFwdThreads / 32) {
            float s = part[threadIdx.x];
#pragma unroll
            for (int o = kFwdThreads / 64; o > 0; o >>= 1) s += __shfl_xor_sync((1u << (kFwdThreads / 32)) - 1u, s, o);
            if (threadIdx.x == 0) atomicAdd(loss_sum, s);
        }
    }
}

// Per-axis gather tables: for every SOURCE index the (few) output indices whose bilinear footprint covers it, with their
// weights.  Built once per call by one thread per source index, each candidate tested with the forward's own arithmetic
// (src_of), so the backward is the exact transpose of the forward.  K entries per source index.
__global__ void __launch_bounds__(128) resize_tables_kernel(int n_src, int n_out, float r, int K, int* __restrict__ cnt,
                                                            int* __restrict__ idx, float* __restrict__ wgt) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_src) return;
    int lo, hi;
    if (r <= 0.f) {  // n_out == 1: the single output samples source 0
        lo = 0;
        hi = (s == 0) ? 0 : -1;
    } else {         // src = r * o in (s - 1, s + 1): conservative integer range
        lo = max(0, (int)floorf((float)(s - 1) / r) - 1);
        hi = min(n_out - 1, (int)ceilf((float)(s + 1) / r) + 1);
    }
    int n = 0;
    for (int o = lo; o <= hi && n < K; o++) {
        int i0, i1;
        float l0, l1;
        src_of(o, r, n_src, i0, i1, l0, l1);
        const float w = (i0 == s ? l0 : 0.f) + (i1 == s ? l1 : 0.f);
        if (w != 0.f) {
            idx[(size_t)s * K + n] = o;
            wgt[(size_t)s * K + n] = w;
            n++;
        }
    }
    cnt[s] = n;
}

struct GatherTables {
    const int* cnt_y; const int* idx_y; const float* w_y;
    const int* cnt_x; const int* idx_x; const float* w_x;
    int Ky, Kx;
};

// grid = (ceil(W / 1024), ceil(C * H / kRowsPerBlock)): a thread owns four consecutive pixels (one 128-bit store) of
// kRowsPerBlock consecutive gradient rows, its x-table entries stay in registers across the rows, the rows' y-table entries
// are block-uniform, and nothing is divided per element.  (History: a flat 64-bit index with % W, % H per element took
// 2.0 ms at config 3; one element per thread in 524 K tiny blocks was block-dispatch bound at 1.4 ms; this form streams.)
constexpr int kRowsPerBlock = 8;   // at least; more when C * H / 8 would exceed the 65535 limit of gridDim.y
constexpr int kMaxKx = 6;   // x-table entries kept in registers; wider tables (strong up-sampling) take the generic loop

__global__ void __launch_bounds__(256) resize_bwd_kernel(ResizeGeom g, GatherTables t, const float* __restrict__ dout,
                                                         float* __restrict__ dfm, int rows_per_block) {
    const int x0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    if (x0 >= g.W) return;
    const int rows = g.C * g.H;
    int nx[4], ix[4][kMaxKx];
    float wx[4][kMaxKx];
    const bool small = t.Kx <= kMaxKx;
    int nmax = 0;  // entries actually present for this thread's four pixels (<= 2 when down-sampling)
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int x = x0 + j;
        nx[j] = x < g.W ? t.cnt_x[x] : 0;
        nmax = max(nmax, nx[j]);
        if (small) {
#pragma unroll
            for (int b = 0; b < kMaxKx; b++) {
                const bool on = b < nx[j];
                ix[j][b] = on ? t.idx_x[(size_t)x * t.Kx + b] : 0;
                wx[j][b] = on ? t.w_x[(size_t)x * t.Kx + b] : 0.f;
            }
        }
    }
    for (int r = 0; r < rows_per_block; r++) {
        const int row = blockIdx.y * rows_per_block + r;  // c * H + y
        if (row >= rows) break;
        const int c = row / g.H, y = row - c * g.H;
        const float* p = dout + (size_t)c * g.Hg * g.Wg;
        const int ny = t.cnt_y[y];
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int a = 0; a < ny; a++) {
            const float* orow = p + (size_t)t.idx_y[(size_t)y * t.Ky + a] * g.Wg;
            const float wy = t.w_y[(size_t)y * t.Ky + a];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                float s = 0.f;
                if (small) {
#pragma unroll
                    for (int b = 0; b < kMaxKx; b++)
                        if (b < nmax) s += wx[j][b] * __ldg(orow + ix[j][b]);  // padded entries: weight 0, index 0
                } else {
                    const int x = x0 + j;
                    for (int b = 0; b < nx[j]; b++) s += t.w_x[(size_t)x * t.Kx + b] * __ldg(orow + t.idx_x[(size_t)x * t.Kx + b]);
                }
                acc[j] += wy * s;
            }
        }
        float* o = dfm + (size_t)row * g.W + x0;
        if (x0 + 3 < g.W && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
            *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (x0 + j < g.W) o[j] = acc[j];
        }
    }
}

// Down-sampling by more than 2 (the reference's 1/2.25 teacher maps): consecutive outputs sample source positions more than
// two apart, so every source pixel has AT MOST ONE output per axis and the gather is a single product.  A block owns
// rows_per_block gradient rows (their y entries staged once in shared memory) and 4 x blockDim columns; a thread's four
// pixels are blockDim apart, so every load and store instruction of a warp covers 128 contiguous bytes whatever W's
// alignment is, and the four rows of a trip are independent loads in flight.
constexpr int kOneMaxRows = 32;

__global__ void __launch_bounds__(512) resize_bwd_one_kernel(ResizeGeom g, GatherTables t, const float* __restrict__ dout,
                                                             float* __restrict__ dfm, int rows_per_block) {
    __shared__ size_t s_off[kOneMaxRows];
    __shared__ float s_wy[kOneMaxRows];
    const int rows = g.C * g.H, row0 = blockIdx.y * rows_per_block, T = blockDim.x;
    if ((int)threadIdx.x < rows_per_block) {
        const int row = row0 + threadIdx.x;
        size_t off = 0;
        float wy = 0.f;
        if (row < rows) {
            const int c = row / g.H, y = row - c * g.H;
            const bool on = t.cnt_y[y] > 0;
            wy = on ? t.w_y[(size_t)y * t.Ky] : 0.f;
            off = ((size_t)c * g.Hg + (on ? t.idx_y[(size_t)y * t.Ky] : 0)) * g.Wg;
        }
        s_off[threadIdx.x] = off;
        s_wy[threadIdx.x] = wy;
    }
    __syncthreads();
    int ix[4];
    float wx[4];
    bool in[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int x = (blockIdx.x * 4 + j) * T + threadIdx.x;
        in[j] = x < g.W;
        const bool on = in[j] && t.cnt_x[x] > 0;
        ix[j] = on ? t.idx_x[(size_t)x * t.Kx] : 0;
        wx[j] = on ? t.w_x[(size_t)x * t.Kx] : 0.f;
    }
    const int nrow = min(rows_per_block, rows - row0);
    for (int r = 0; r < nrow; r += 4) {
        float v[4][4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const bool live = r + u < nrow;
            const float wy = live ? s_wy[r + u] : 0.f;
            const float* orow = dout + (live ? s_off[r + u] : 0);
#pragma unroll
            for (int j = 0; j < 4; j++) v[u][j] = (wy != 0.f) ? wy * wx[j] * __ldg(orow + ix[j]) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            if (r + u >= nrow) break;
            float* o = dfm + (size_t)(row0 + r + u) * g.W + (size_t)blockIdx.x * 4 * T + threadIdx.x;
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (in[j]) o[j * T] = v[u][j];
        }
    }
}

ResizeGeom make_geom(int C, int H, int W, int Hg, int Wg) {
    ResizeGeom g;
    g.C = C; g.H = H; g.W = W; g.Hg = Hg; g.Wg = Wg;
    g.ry = Hg > 1 ? (float)(H - 1) / (float)(Hg - 1) : 0.f;
    g.rx = Wg > 1 ? (float)(W - 1) / (float)(Wg - 1) : 0.f;
    return g;
}

}  // namespace

template <typename GT>
cudaError_t launch_feature_resize_fwd(int C, int H, int W, int Hg, int Wg, const float* fm, const GT* gt, float grad_scale,
                                      float* out, float* loss_sum, cudaStream_t s) {
    const size_t n = (size_t)C * Hg * Wg;
    if (n == 0) return cudaSuccess;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t rows = (size_t)C * Hg;
    if (rows > 0x7fffffffu) return cudaErrorInvalidValue;
    const unsigned grid = (unsigned)std::min<size_t>((rows + kFwdThreads / 32 - 1) / (kFwdThreads / 32), (size_t)sms * 8);
    resize_fwd_kernel<GT><<<grid, kFwdThreads, 0, s>>>(make_geom(C, H, W, Hg, Wg), fm, gt, grad_scale, out, loss_sum);
    g_launches++;
    return cudaGetLastError();
}
template cudaError_t launch_feature_resize_fwd(int, int, int, int, int, const float*, const float*, float, float*, float*,
                                               cudaStream_t);
template cudaError_t launch_feature_resize_fwd(int, int, int, int, int, const float*, const __half*, float, float*,
                                               float*, cudaStream_t);

cudaError_t launch_feature_resize_bwd(int C, int H, int W, int Hg, int Wg, const float* dout, float* dfm, cudaStream_t s) {
    const size_t n = (size_t)C * H * W;
    if (n == 0) return cudaSuccess;
    const ResizeGeom g = make_geom(C, H, W, Hg, Wg);
    auto cap = [](float r, int n_out) { return r > 0.f ? std::min(n_out, (int)std::ceil(2.0f / r) + 3) : 1; };
    const int Ky = cap(g.ry, Hg), Kx = cap(g.rx, Wg);
    // tables: cnt[H] idx[H*Ky] w[H*Ky] cnt[W] idx[W*Kx] w[W*Kx], stream-ordered scratch (pool-cached after the first call)
    const size_t words = (size_t)H * (1 + 2 * Ky) + (size_t)W * (1 + 2 * Kx);
    int* ws = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&ws, words * 4, s);
    if (e != cudaSuccess) return e;
    GatherTables t;
    int* q = ws;
    t.cnt_y = q; q += H; t.idx_y = q; q += (size_t)H * Ky; t.w_y = reinterpret_cast<float*>(q); q += (size_t)H * Ky;
    t.cnt_x = q; q += W; t.idx_x = q; q += (size_t)W * Kx; t.w_x = reinterpret_cast<float*>(q);
    t.Ky = Ky; t.Kx = Kx;
    resize_tables_kernel<<<(H + 127) / 128, 128, 0, s>>>(H, Hg, g.ry, Ky, const_cast<int*>(t.cnt_y), const_cast<int*>(t.idx_y),
                                                      const_cast<float*>(t.w_y));
    resize_tables_kernel<<<(W + 127) / 128, 128, 0, s>>>(W, Wg, g.rx, Kx, const_cast<int*>(t.cnt_x), const_cast<int*>(t.idx_x),
                                                      const_cast<float*>(t.w_x));
    const int rows = C * H;
    if (g.ry >= 2.001f && g.rx >= 2.001f && (rows + kOneMaxRows - 1) / kOneMaxRows <= 65535) {
        const int T = std::min(512, ((W + 3) / 4 + 31) / 32 * 32);
        const int rpb = std::max(16, std::min(kOneMaxRows, (rows + 65534) / 65535));
        resize_bwd_one_kernel<<<dim3((W + 4 * T - 1) / (4 * T), (rows + rpb - 1) / rpb), T, 0, s>>>(g, t, dout, dfm, rpb);
    } else {
        const int rpb = std::max(kRowsPerBlock, (rows + 65534) / 65535);
        resize_bwd_kernel<<<dim3((W + 1023) / 1024, (rows + rpb - 1) / rpb), 256, 0, s>>>(g, t, dout, dfm, rpb);
    }
    g_launches += 3;
    e = cudaGetLastError();
    cudaFreeAsync(ws, s);
    return e;
}

}  // namespace f3dgs
