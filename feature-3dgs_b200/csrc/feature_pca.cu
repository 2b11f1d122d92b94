// PCA picture of a feature map: render.py's feature_visualize_saving (render.py:147-180) without the map leaving the
// device.  Shapes: x [C, N] (a map [C,H,W] as N = H W pixels, p = y W + x), float32 or float16.  With
//     xh_p = x_p / max(||x_p||, 1e-12)  (applied as x_p * (1 / max(||x_p||, 1e-12)), the norm summed in fp32)
//     samples s = 0 .. n - 1 are the pixels p = 3 s, n = ceil(N / 3)
// the three calls are
//     moments  pass 1 (tile_kernel<kMoments>): per 32-sample tile the samples' inverse norms (to scratch) and the tile's
//              per-channel sums of xh in fp32, accumulated per CTA in fp64; mean_kernel adds the CTA partials in a
//              fixed order -> mean [C] (fp32).
//              pass 2 (gram_kernel): G = sum_s (xh_s - mean)(xh_s - mean)^T over the upper-triangular 128 x 128 tiles,
//              centred on load (one fma per element), fp32 FMA accumulation over blocks of kGramBlock samples, every
//              block added into the CTA's fp64 partial tile; cov_kernel adds the split partials in a fixed order ->
//              cov [C, C] = G / (n - 1) in fp64, symmetric bitwise.
//     range    t_k = c_k . (xh_s - mean) for every sample and k (tile_kernel<kProject>) -> 3n floats, sorted by
//              cub::DeviceRadixSort, and percentile_kernel interpolates np.percentile(t, [1, 99]) (linear) into range[2]
//              on the device: no host sync.
//     image    one read of the map (tile_kernel<kImage>): per pixel the norm and the three centred dot products,
//              image[p, k] = clamp((t_k - lo) / (hi - lo), 0, 1) (NaN passes through, as torch.clamp).
// A tile is 32 pixels (one per lane) x all C channels, staged in shared memory by 8 warps that each own the channels
// c = warp (mod 8); the loads of a warp are one row of 32 pixels (coalesced at stride 1).  The range and image calls share
// the tile code, so a sample's t in the range call is bitwise the t its pixel gets in the image call.
// No float atomics and fixed summation orders: every output is bitwise reproducible.
#include <cub/cub.cuh>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels.h"
#include "tf32_mma.cuh"

namespace f3dgs {
namespace {

constexpr int kWarps = 8, kThreads = 32 * kWarps;
constexpr int kRow = 33;             // tile row stride in floats (channel-major rows of 32 pixels, padded: no conflicts)
constexpr int kMomentCtas = 1024;    // pass-1 CTAs (fp64 partial means: kMomentCtas x C)
constexpr int kGT = 128;             // Gram tile edge
constexpr int kGK = 16;              // samples per Gram chunk
constexpr int kGS = kGT + 4;         // Gram smem row stride: at most 2-way conflicts on stores with samples fastest
constexpr int kGramBlock = 2048;     // samples per fp32 accumulation block
constexpr int kSms = 132;            // H100 SXM; the Gram kernel runs one CTA per SM (255 registers)

size_t up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

int gram_tiles(int C) {
    const int nt = (C + kGT - 1) / kGT;
    return nt * (nt + 1) / 2;
}
// tiles x splits fills one or two whole waves of kSms CTAs as closely as possible (splits <= blocks <= n)
int gram_splits(int C, int n) {
    const int blocks = (n + kGramBlock - 1) / kGramBlock, T = gram_tiles(C);
    int best = 1;
    double util = 0.0;
    for (int w = 1; w <= 2; w++) {
        const int S = std::max(1, std::min(blocks, kSms * w / T)), ctas = T * S;
        const double u = (double)ctas / (kSms * ((ctas + kSms - 1) / kSms));
        if (u > util + 1e-9) { util = u; best = S; }
    }
    return best;
}
int moment_ctas(int n) { return std::min((n + 31) / 32, kMomentCtas); }

struct PcaLayout {  // scratch of the moments and range calls; every size is a function of (C, N)
    size_t inv, mpart, gpart, keys, sorted, sort_tmp;
    PcaLayout(int C, int N) {
        const size_t n = ((size_t)N + 2) / 3;
        size_t o = 0;
        inv = o;     o = up(o + n * 4);
        mpart = o;   o = up(o + (size_t)moment_ctas((int)n) * C * 8);
        gpart = o;   o = up(o + (size_t)gram_splits(C, (int)n) * gram_tiles(C) * kGT * kGT * 8);
        keys = o;    o = up(o + 3 * n * 4);
        sorted = o;  o = up(o + 3 * n * 4);
        sort_tmp = o;
    }
};

cudaError_t sort_bytes(int m, size_t* bytes) {
    *bytes = 0;
    return cub::DeviceRadixSort::SortKeys(nullptr, *bytes, (const float*)nullptr, (float*)nullptr, m);
}

enum Mode { kMoments, kProject, kImage };

template <typename T>
struct TileArgs {
    int C, N, stride, count;  // pixels p = stride * s for s < count
    const T* x;
    const float* mean;        // [C]     (kProject, kImage)
    const float* comp;        // [3, C]  (kProject, kImage)
    const float* range;       // [2]     (kImage)
    float* inv;               // [count] (kMoments)
    double* mpart;            // [gridDim.x, C] (kMoments)
    float* out;               // keys [3, count] (kProject) or image [N, 3] (kImage)
};

// CTA loops over the 32-pixel tiles blockIdx.x, blockIdx.x + gridDim.x, ... in that fixed order
template <Mode M, typename T>
__global__ void __launch_bounds__(kThreads) tile_kernel(TileArgs<T> a) {
    extern __shared__ float xs[];                // [C][kRow]
    __shared__ float red[3][kWarps][32];
    __shared__ float inv_s[32];
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, C = a.C;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};        // kMoments: channels threadIdx.x + 256 j (C <= 1024)
    const int tiles = (a.count + 31) / 32;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int s = tile * 32 + l;
        const bool in = s < a.count;
        const T* px = a.x + (size_t)a.stride * (in ? s : 0);
        float ss = 0.f;
#pragma unroll 16  // 16 loads in flight per thread: the pass is bound by bytes in flight
        for (int c = w; c < C; c += kWarps) {
            const float v = in ? load_f32(px + (size_t)c * a.N) : 0.f;
            xs[c * kRow + l] = v;
            ss = fmaf(v, v, ss);
        }
        red[0][w][l] = ss;
        __syncthreads();
        if (w == 0) {
            float t = 0.f;
#pragma unroll
            for (int i = 0; i < kWarps; i++) t += red[0][i][l];
            const float iv = 1.f / fmaxf(sqrtf(t), 1e-12f);
            inv_s[l] = iv;
            if constexpr (M == kMoments)
                if (in) a.inv[s] = iv;
        }
        __syncthreads();
        if constexpr (M == kMoments) {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int c = threadIdx.x + kThreads * j;
                if (c < C) {
                    float t = 0.f;
                    for (int i = 0; i < 32; i++) t = fmaf(xs[c * kRow + i], inv_s[i], t);  // zero past count
                    acc[j] += (double)t;
                }
            }
        } else {
            const float iv = inv_s[l];
            float d0 = 0.f, d1 = 0.f, d2 = 0.f;
#pragma unroll 4
            for (int c = w; c < C; c += kWarps) {
                const float v = fmaf(xs[c * kRow + l], iv, -__ldg(a.mean + c));
                d0 = fmaf(__ldg(a.comp + c), v, d0);
                d1 = fmaf(__ldg(a.comp + C + c), v, d1);
                d2 = fmaf(__ldg(a.comp + 2 * C + c), v, d2);
            }
            red[0][w][l] = d0; red[1][w][l] = d1; red[2][w][l] = d2;
            __syncthreads();
            if (w < 3 && in) {
                float t = 0.f;
#pragma unroll
                for (int i = 0; i < kWarps; i++) t += red[w][i][l];
                if constexpr (M == kProject) {
                    a.out[(size_t)w * a.count + s] = t;
                } else {
                    const float lo = __ldg(a.range), hi = __ldg(a.range + 1);
                    const float v = (t - lo) / (hi - lo);
                    a.out[(size_t)s * 3 + w] = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
                }
            }
        }
        __syncthreads();  // xs, red and inv_s are rewritten by the next tile
    }
    if constexpr (M == kMoments) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int c = threadIdx.x + kThreads * j;
            if (c < C) a.mpart[(size_t)blockIdx.x * C + c] = acc[j];
        }
    }
}

__global__ void mean_kernel(int C, int n, int parts, const double* __restrict__ mpart, float* __restrict__ mean) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double t = 0.0;
    for (int b = 0; b < parts; b++) t += mpart[(size_t)b * C + c];
    mean[c] = (float)(t / n);
}

template <typename T>
struct GramArgs {
    int C, N, n, nt, splits;
    const T* x;
    const float* inv;    // [n]
    const float* mean;   // [C]
    double* gpart;       // [splits][tiles][kGT * kGT]
};

// CTA (tile, split): the upper-triangular tile (I, J), I <= J, over the split's contiguous sample range
// [n split / splits, n (split + 1) / splits) in blocks of kGramBlock.  256 threads; thread (ty, tx) = (t / 16, t % 16)
// owns rows {4 ty .. 4 ty + 3, 64 + 4 ty ..} x the same columns of tx.
template <typename T>
__global__ void __launch_bounds__(kThreads, 1) gram_kernel(GramArgs<T> a) {
    __shared__ __align__(16) float As[2][kGK][kGS];
    __shared__ __align__(16) float Bs[2][kGK][kGS];
    int I = 0, J = blockIdx.x;
    while (J >= a.nt - I) { J -= a.nt - I; I++; }
    J += I;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    // loader: chunk slot ls = tid % 16, channels lc + 16 i (i < 8) of both operands
    constexpr int kL = kGT * kGK / kThreads;
    const int ls = tid & 15, lc = tid >> 4;
    const int ci0 = I * kGT + lc, cj0 = J * kGT + lc;
    float ra[kL], rb[kL], rinv = 0.f;
    bool rin = false;
    auto fetch = [&](int s, int end) {  // raw x of sample s (0 past end or C)
        rin = s < end;
        const T* px = a.x + (size_t)3 * (rin ? s : 0);
        rinv = rin ? __ldg(a.inv + s) : 0.f;
#pragma unroll
        for (int i = 0; i < kL; i++) {
            const int ci = ci0 + 16 * i, cj = cj0 + 16 * i;
            ra[i] = rin && ci < a.C ? load_f32(px + (size_t)ci * a.N) : 0.f;
            rb[i] = rin && cj < a.C ? load_f32(px + (size_t)cj * a.N) : 0.f;
        }
    };
    auto store = [&](int buf) {  // centred on store: xh - mean, exactly 0 past the range or C
#pragma unroll
        for (int i = 0; i < kL; i++) {
            const int ci = ci0 + 16 * i, cj = cj0 + 16 * i;
            As[buf][ls][lc + 16 * i] = rin && ci < a.C ? fmaf(ra[i], rinv, -__ldg(a.mean + ci)) : 0.f;
            Bs[buf][ls][lc + 16 * i] = rin && cj < a.C ? fmaf(rb[i], rinv, -__ldg(a.mean + cj)) : 0.f;
        }
    };
    double* part = a.gpart + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * kGT * kGT;
    const int lo = (int)((int64_t)a.n * blockIdx.y / a.splits), hi = (int)((int64_t)a.n * (blockIdx.y + 1) / a.splits);
    bool first = true;
    for (int s0 = lo; s0 < hi; s0 += kGramBlock) {
        const int end = min(s0 + kGramBlock, hi), chunks = (end - s0 + kGK - 1) / kGK;
        float acc[8][8];
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
            for (int j = 0; j < 8; j++) acc[i][j] = 0.f;
        fetch(s0 + ls, end);
        store(0);
        __syncthreads();
        for (int ch = 0; ch < chunks; ch++) {
            const int buf = ch & 1;
            if (ch + 1 < chunks) fetch(s0 + (ch + 1) * kGK + ls, end);
#pragma unroll
            for (int k = 0; k < kGK; k++) {
                const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][4 * ty]);
                const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + 4 * ty]);
                const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][4 * tx]);
                const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + 4 * tx]);
                const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int i = 0; i < 8; i++)
#pragma unroll
                    for (int j = 0; j < 8; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
            }
            if (ch + 1 < chunks) store(buf ^ 1);
            __syncthreads();
        }
        // the block's fp32 sums into this CTA's fp64 partial (its own slot: no atomics)
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int r = (i < 4 ? 0 : 64) + 4 * ty + (i & 3);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const int c = (j < 4 ? 0 : 64) + 4 * tx + (j & 3);
                double* d = part + r * kGT + c;
                *d = first ? (double)acc[i][j] : *d + (double)acc[i][j];
            }
        }
        first = false;  // splits <= n: every range is non-empty, so every slot is written
    }
}

// cov[i, j] = cov[j, i] = (sum over splits of G[min, max]) / (n - 1), the splits added in order
__global__ void cov_kernel(int C, int n, int nt, int tiles, int splits, const double* __restrict__ gpart,
                           double* __restrict__ cov) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)C * C) return;
    const int r = (int)(e / C), c = (int)(e - (size_t)r * C);
    const int i = min(r, c), j = max(r, c), I = i / kGT, J = j / kGT;
    const int tile = I * nt - I * (I - 1) / 2 + (J - I);
    const double* p = gpart + (size_t)tile * kGT * kGT + (i - I * kGT) * kGT + (j - J * kGT);
    double t = 0.0;
    for (int sp = 0; sp < splits; sp++) t += p[(size_t)sp * tiles * kGT * kGT];
    cov[e] = t / (n - 1);
}

// np.percentile(v, q, method='linear') of the m sorted values for q = 1 and 99, numpy's own lerp
__global__ void percentile_kernel(int m, const float* __restrict__ v, float* __restrict__ range) {
    const double qs[2] = {0.01, 0.99};
    for (int k = 0; k < 2; k++) {
        const double h = (double)(m - 1) * qs[k];
        const int j = min((int)floor(h), m - 1), j1 = min(j + 1, m - 1);
        const double t = h - j, a = v[j], b = v[j1], d = b - a;
        range[k] = (float)(t >= 0.5 ? b - d * (1.0 - t) : a + d * t);
    }
}

template <Mode M, typename T>
cudaError_t launch_tile(const TileArgs<T>& a, unsigned grid, cudaStream_t s) {
    const size_t smem = (size_t)a.C * kRow * 4;
    cudaError_t e = cudaFuncSetAttribute(tile_kernel<M, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    tile_kernel<M, T><<<grid, kThreads, smem, s>>>(a);
    g_launches++;
    return cudaGetLastError();
}

template <typename T>
cudaError_t moments_run(int C, int N, const T* x, char* scratch, float* mean, double* cov, cudaStream_t s) {
    const PcaLayout ly(C, N);
    const int n = (N + 2) / 3, parts = moment_ctas(n);
    float* inv = reinterpret_cast<float*>(scratch + ly.inv);
    double* mpart = reinterpret_cast<double*>(scratch + ly.mpart);
    TileArgs<T> ta{};
    ta.C = C; ta.N = N; ta.stride = 3; ta.count = n;
    ta.x = x; ta.inv = inv; ta.mpart = mpart;
    cudaError_t e = launch_tile<kMoments>(ta, (unsigned)parts, s);
    if (e != cudaSuccess) return e;
    mean_kernel<<<(C + 255) / 256, 256, 0, s>>>(C, n, parts, mpart, mean);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    GramArgs<T> ga;
    ga.C = C; ga.N = N; ga.n = n;
    ga.nt = (C + kGT - 1) / kGT;
    ga.splits = gram_splits(C, n);
    ga.x = x; ga.inv = inv; ga.mean = mean;
    ga.gpart = reinterpret_cast<double*>(scratch + ly.gpart);
    const int tiles = gram_tiles(C);
    gram_kernel<T><<<dim3((unsigned)tiles, (unsigned)ga.splits), kThreads, 0, s>>>(ga);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const size_t cc = (size_t)C * C;
    cov_kernel<<<(unsigned)((cc + 255) / 256), 256, 0, s>>>(C, n, ga.nt, tiles, ga.splits, ga.gpart, cov);
    g_launches++;
    return cudaGetLastError();
}

template <typename T>
cudaError_t range_run(int C, int N, const T* x, const float* mean, const float* comp, char* scratch, float* range,
                      cudaStream_t s) {
    const PcaLayout ly(C, N);
    const int n = (N + 2) / 3, m = 3 * n;
    float* keys = reinterpret_cast<float*>(scratch + ly.keys);
    float* sorted = reinterpret_cast<float*>(scratch + ly.sorted);
    TileArgs<T> ta{};
    ta.C = C; ta.N = N; ta.stride = 3; ta.count = n;
    ta.x = x; ta.mean = mean; ta.comp = comp; ta.out = keys;
    cudaError_t e = launch_tile<kProject>(ta, (unsigned)((n + 31) / 32), s);
    if (e != cudaSuccess) return e;
    size_t sb = 0;
    if ((e = sort_bytes(m, &sb)) != cudaSuccess) return e;
    if ((e = cub::DeviceRadixSort::SortKeys(scratch + ly.sort_tmp, sb, keys, sorted, m, 0, 32, s)) != cudaSuccess)
        return e;
    percentile_kernel<<<1, 1, 0, s>>>(m, sorted, range);
    g_launches++;
    return cudaGetLastError();
}

template <typename T>
cudaError_t image_run(int C, int N, const T* x, const float* mean, const float* comp, const float* range, float* image,
                      cudaStream_t s) {
    TileArgs<T> ta{};
    ta.C = C; ta.N = N; ta.stride = 1; ta.count = N;
    ta.x = x; ta.mean = mean; ta.comp = comp; ta.range = range; ta.out = image;
    return launch_tile<kImage>(ta, (unsigned)((N + 31) / 32), s);
}

}  // namespace

size_t pca_scratch_fixed_bytes(int C, int N) { return PcaLayout(C, N).sort_tmp; }

cudaError_t pca_scratch_bytes(int C, int N, size_t* bytes) {
    *bytes = 0;
    size_t sb = 0;
    const cudaError_t e = sort_bytes(3 * ((N + 2) / 3), &sb);
    if (e != cudaSuccess) return e;
    *bytes = PcaLayout(C, N).sort_tmp + up(sb);
    return cudaSuccess;
}

cudaError_t launch_pca_moments(int C, int N, const float* x, char* scratch, float* mean, double* cov, cudaStream_t s) {
    return moments_run(C, N, x, scratch, mean, cov, s);
}
cudaError_t launch_pca_moments(int C, int N, const __half* x, char* scratch, float* mean, double* cov, cudaStream_t s) {
    return moments_run(C, N, x, scratch, mean, cov, s);
}
cudaError_t launch_pca_range(int C, int N, const float* x, const float* mean, const float* comp, char* scratch,
                             float* range, cudaStream_t s) {
    return range_run(C, N, x, mean, comp, scratch, range, s);
}
cudaError_t launch_pca_range(int C, int N, const __half* x, const float* mean, const float* comp, char* scratch,
                             float* range, cudaStream_t s) {
    return range_run(C, N, x, mean, comp, scratch, range, s);
}
cudaError_t launch_pca_image(int C, int N, const float* x, const float* mean, const float* comp, const float* range,
                             float* image, cudaStream_t s) {
    return image_run(C, N, x, mean, comp, range, image, s);
}
cudaError_t launch_pca_image(int C, int N, const __half* x, const float* mean, const float* comp, const float* range,
                             float* image, cudaStream_t s) {
    return image_run(C, N, x, mean, comp, range, image, s);
}

}  // namespace f3dgs
