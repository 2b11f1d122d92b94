// 1x1-convolution feature decoder of the reference's --speedup mode, fused with the L1 feature loss and its gradients.
// Reference: models/networks.py:107-119 (CNN_decoder = nn.Conv2d(Cin, Cout, kernel_size=1) with bias), train.py:100-104
//     feature_map = cnn_decoder(resized_feature_map);  Ll1_feature = l1_loss(feature_map, gt_feature_map)
// Shapes: x [Cin, N] (the resized map, N = Hg * Wg), W [Cout, Cin], b [Cout], gt [Cout, N].
//     decode  y = W x + b                                              -> [Cout, N]
//     loss    s = sign(y - gt) (sign(0) = 0);  loss_sum = sum |y - gt|;  dL/dx = gs W^T s  (written);
//             dL/dW += gs s x^T;  dL/db += gs sum_n s                  (gs = grad_scale = loss_weight / (Cout N))
// In PyTorch the loss is a GEMM writing y, an L1 reading y and gt, a sign kernel writing a Cout x N gradient, and two
// more GEMMs reading that gradient back.  Here y and s never reach DRAM as fp32:
//     prep     rounds W to TF32 and zero-pads it to [Cout_pad, Cp] (Cp = 8 KT >= Cin), pads b to Cout_pad.
//     kernel A a warp owns 16 pixels and walks Cout in steps of 32 output channels (W streamed through shared memory by
//              cp.async, double-buffered).  Per step:  Y^T[16 px, 32] = X^T W^T (TF32 mma.sync m16n8k8, fp32 accumulate,
//              bias as the initial accumulator), then in loss mode s and |y - gt| straight from the accumulator
//              registers, and  dX^T[16 px, Cin] += S^T W  with S^T taken from the same registers: the accumulator of
//              m16n8k8 holds columns (2t, 2t + 1) where the A operand wants (t, t + 4), so the k index of the second
//              product is permuted (slot t <-> channel 2t, slot t + 4 <-> 2t + 1) on both operands.  The signs are
//              also written as one 32-bit word per (output channel, 16 pixels): 16 non-zero bits, 16 negative bits.
//     kernel B dW = s x^T and the sign counts for db, split-K over pixel ranges into per-split partials (s from the bit
//              words, x rounded to TF32; the same slot permutation puts a thread's two pixels side by side).
//     finish   sums the split partials in a fixed order and ADDS gs * (sum) into dW and db; a one-CTA kernel sums the
//              per-CTA loss partials of kernel A in double.
// No float atomics: every output element is written by one thread and every sum has a fixed order, so results are
// bitwise reproducible.  Decode and loss mode run the same code for y, so decode(x) as gt gives exactly zero loss.
// gt (loss) and y (decode) may also be float16, the data format's teacher maps: a float16 gt is upcast exactly at its load
// (the result is the float32 one for gt.float()), a float16 y is rounded to nearest even at its store (y.half()).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels.h"
#include "tf32_mma.cuh"

namespace f3dgs {
namespace {

constexpr int kWarpsA = 8, kThreadsA = 32 * kWarpsA;
constexpr int kPixWarp = 16;                   // pixels per warp: the M = 16 rows of one mma tile
constexpr int kWarpsB = 4, kThreadsB = 32 * kWarpsB;
constexpr int kCoutB = 32 * kWarpsB;           // output channels per CTA of kernel B (32 per warp)
constexpr int kCinB = 32;                      // input channels per CTA of kernel B
constexpr int kCoutAlign = kCoutB;             // Cout_pad: a whole number of kernel B tiles (and of kernel A steps)
constexpr int kTargetCtasB = 1024;             // split-K: about this many kernel B CTAs whatever the shape
constexpr int kReduceThreads = 512;

// sign as a TF32 operand: +1, -1 or 0 (exact)
__device__ __forceinline__ uint32_t sign_bits(float d) { return d > 0.f ? 0x3f800000u : (d < 0.f ? 0xbf800000u : 0u); }
// the sign of pixel i (0..15) of a bit word
__device__ __forceinline__ uint32_t word_sign(uint32_t w, int i) {
    return (((w >> i) & 1u) * 0x3f800000u) | (((w >> (16 + i)) & 1u) << 31);
}

__device__ __forceinline__ void store_f32(float* p, float v) { *p = v; }
__device__ __forceinline__ void store_f32(__half* p, float v) { *p = __float2half_rn(v); }

template <typename T>      // element type of gt and y: float or __half
struct DecArgs {
    int Cin, Cout, N, N16;
    const float* wt;       // [Cout_pad, Cp] TF32, zero-padded
    const float* bias;     // [Cout_pad], zero-padded
    const float* x;        // [Cin, N]
    const T* gt;           // [Cout, N]            (loss)
    T* y;                  // [Cout, N]            (decode)
    float* dx;             // [Cin, N]             (loss)
    uint32_t* bits;        // [Cout, N16]          (loss)
    float* loss_part;      // [gridDim.x]          (loss)
    float grad_scale;
};

template <int KT>
struct DecSmem {
    static constexpr int Cp = 8 * KT, SW = Cp + 4;  // W rows padded by 4 floats: conflict-free fragment loads
    static constexpr bool x_in_regs = KT <= 16;     // Cin <= 128: X^T fragments in registers, else in shared memory
    // Cin > 128: two warps share a 16-pixel tile, both form Y and each accumulates half of dX (128 registers would spill)
    static constexpr int share = x_in_regs ? 1 : 2;
    static constexpr int dkt = KT / share;          // n8 tiles of dX per warp
    static constexpr int step = x_in_regs ? 32 : 16;  // output channels per step
    static constexpr size_t bytes = (size_t)2 * step * SW * 4 + (x_in_regs ? 0 : (size_t)kWarpsA * KT * 32 * 16);
};

template <int KT, bool LOSS, typename T>
__global__ void __launch_bounds__(kThreadsA, 1) decoder_kernel(DecArgs<T> a) {
    using S = DecSmem<KT>;
    constexpr int Cp = S::Cp, SW = S::SW, kStep = S::step, kNT = kStep / 8;  // kNT n8 tiles of Y = k8 steps of dX
    extern __shared__ float4 smem4[];
    float* ws = reinterpret_cast<float*>(smem4);                     // [2][kStep][SW]
    float4* xs = smem4 + (2 * kStep * SW) / 4 + threadIdx.x / 32 * KT * 32;  // this warp's [KT][32] fragments
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int N = a.N, Cin = a.Cin, Cout = a.Cout;
    const int blk = blockIdx.x * (kWarpsA / S::share) + warp / S::share;  // 16-pixel block of this warp
    const int part = warp % S::share, kt0 = part * S::dkt;                  // its dX tiles: kt0 .. kt0 + dkt - 1
    const int pa = blk * kPixWarp + g, pb = pa + 8;
    const bool ina = pa < N, inb = pb < N;
    const int steps = (Cout + kStep - 1) / kStep;

    auto load_w = [&](int st) {
        const float* src = a.wt + (size_t)st * kStep * Cp;
        float* dst = ws + (st & 1) * kStep * SW;
        for (int i = threadIdx.x; i < kStep * Cp / 4; i += kThreadsA) {
            const int r = i / (Cp / 4), c = (i - r * (Cp / 4)) * 4;
            cp_async16(dst + r * SW + c, src + (size_t)r * Cp + c);
        }
        cp_async_commit();
    };
    load_w(0);

    // X^T A-fragments (pixel, input channel), rounded to TF32, zero outside the image and past Cin
    uint32_t xr[S::x_in_regs ? KT : 1][4];
#pragma unroll
    for (int kt = 0; kt < KT; kt++) {
        const int c0 = 8 * kt + t, c1 = c0 + 4;
        uint32_t f[4];
        f[0] = to_tf32(c0 < Cin && ina ? __ldg(a.x + (size_t)c0 * N + pa) : 0.f);
        f[1] = to_tf32(c0 < Cin && inb ? __ldg(a.x + (size_t)c0 * N + pb) : 0.f);
        f[2] = to_tf32(c1 < Cin && ina ? __ldg(a.x + (size_t)c1 * N + pa) : 0.f);
        f[3] = to_tf32(c1 < Cin && inb ? __ldg(a.x + (size_t)c1 * N + pb) : 0.f);
        if constexpr (S::x_in_regs) {
#pragma unroll
            for (int i = 0; i < 4; i++) xr[kt][i] = f[i];
        } else {
            xs[kt * 32 + lane] = make_float4(__uint_as_float(f[0]), __uint_as_float(f[1]), __uint_as_float(f[2]),
                                             __uint_as_float(f[3]));
        }
    }

    float dacc[LOSS ? S::dkt : 1][4];  // dX^T (pixel, input channel) tiles
#pragma unroll
    for (int nt = 0; nt < (LOSS ? S::dkt : 1); nt++)
#pragma unroll
        for (int i = 0; i < 4; i++) dacc[nt][i] = 0.f;
    float lsum = 0.f;

    for (int st = 0; st < steps; st++) {
        cp_async_wait_all();
        __syncthreads();  // chunk st has landed, and every warp is done with the buffer chunk st + 1 overwrites
        if (st + 1 < steps) load_w(st + 1);
        const float* w = ws + (st & 1) * kStep * SW;
        const int co = st * kStep;

        // targets: issued before the products they wait for, except at Cin > 128 where the registers go to dX
        float gv[kNT][4];
        auto load_gt = [&]() {
#pragma unroll
            for (int n = 0; n < kNT; n++) {
                const int c = co + 8 * n + 2 * t;
                const bool va = c < Cout, vb = c + 1 < Cout;
                gv[n][0] = va && ina ? load_f32(a.gt + (size_t)c * N + pa) : 0.f;
                gv[n][1] = vb && ina ? load_f32(a.gt + (size_t)(c + 1) * N + pa) : 0.f;
                gv[n][2] = va && inb ? load_f32(a.gt + (size_t)c * N + pb) : 0.f;
                gv[n][3] = vb && inb ? load_f32(a.gt + (size_t)(c + 1) * N + pb) : 0.f;
            }
        };
        if constexpr (LOSS && S::x_in_regs) load_gt();

        // Y^T tiles (pixel g / g + 8, output channel 2t / 2t + 1 of n-tile n), bias as the initial accumulator
        float yv[kNT][4];
#pragma unroll
        for (int n = 0; n < kNT; n++) {
            const float b0 = __ldg(a.bias + co + 8 * n + 2 * t), b1 = __ldg(a.bias + co + 8 * n + 2 * t + 1);
            yv[n][0] = b0; yv[n][1] = b1; yv[n][2] = b0; yv[n][3] = b1;
        }
#pragma unroll
        for (int kt = 0; kt < KT; kt++) {
            uint32_t af[4];
            if constexpr (S::x_in_regs) {
#pragma unroll
                for (int i = 0; i < 4; i++) af[i] = xr[kt][i];
            } else {
                const float4 v = xs[kt * 32 + lane];
                af[0] = __float_as_uint(v.x); af[1] = __float_as_uint(v.y);
                af[2] = __float_as_uint(v.z); af[3] = __float_as_uint(v.w);
            }
#pragma unroll
            for (int n = 0; n < kNT; n++) {
                const float* wr = w + (8 * n + g) * SW + 8 * kt + t;
                mma_tf32(yv[n], af, __float_as_uint(wr[0]), __float_as_uint(wr[4]));
            }
        }

        if constexpr (!LOSS) {
            if (part != 0) continue;  // the other warp of the pair stores the same y
#pragma unroll
            for (int n = 0; n < kNT; n++) {
                const int c = co + 8 * n + 2 * t;
                if (c < Cout) {
                    if (ina) store_f32(a.y + (size_t)c * N + pa, yv[n][0]);
                    if (inb) store_f32(a.y + (size_t)c * N + pb, yv[n][2]);
                }
                if (c + 1 < Cout) {
                    if (ina) store_f32(a.y + (size_t)(c + 1) * N + pa, yv[n][1]);
                    if (inb) store_f32(a.y + (size_t)(c + 1) * N + pb, yv[n][3]);
                }
            }
        } else {
            if constexpr (!S::x_in_regs) load_gt();
            uint32_t sf[kNT][4];  // S^T A-fragments: (pixel g / g + 8, k slot t <-> channel 2t, slot t + 4 <-> 2t + 1)
#pragma unroll
            for (int n = 0; n < kNT; n++) {
                const int c = co + 8 * n + 2 * t;
                const bool va = c < Cout, vb = c + 1 < Cout;
                const float d0 = va && ina ? yv[n][0] - gv[n][0] : 0.f;  // (pixel g,     channel c)
                const float d1 = vb && ina ? yv[n][1] - gv[n][1] : 0.f;  // (pixel g,     channel c + 1)
                const float d2 = va && inb ? yv[n][2] - gv[n][2] : 0.f;  // (pixel g + 8, channel c)
                const float d3 = vb && inb ? yv[n][3] - gv[n][3] : 0.f;  // (pixel g + 8, channel c + 1)
                if (part == 0) lsum += (fabsf(d0) + fabsf(d1)) + (fabsf(d2) + fabsf(d3));
                // bit words of channels c and c + 1 for the warp's 16 pixels, OR-combined over the 8 lanes sharing t
                uint32_t w0 = ((uint32_t)(d0 != 0.f) << g) | ((uint32_t)(d2 != 0.f) << (g + 8)) |
                              ((uint32_t)(d0 < 0.f) << (g + 16)) | ((uint32_t)(d2 < 0.f) << (g + 24));
                uint32_t w1 = ((uint32_t)(d1 != 0.f) << g) | ((uint32_t)(d3 != 0.f) << (g + 8)) |
                              ((uint32_t)(d1 < 0.f) << (g + 16)) | ((uint32_t)(d3 < 0.f) << (g + 24));
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                    w0 |= __shfl_xor_sync(0xffffffffu, w0, o);
                    w1 |= __shfl_xor_sync(0xffffffffu, w1, o);
                }
                if (g == 0 && part == 0 && blk < a.N16) {
                    if (va) a.bits[(size_t)c * a.N16 + blk] = w0;
                    if (vb) a.bits[(size_t)(c + 1) * a.N16 + blk] = w1;
                }
                sf[n][0] = sign_bits(d0); sf[n][1] = sign_bits(d2); sf[n][2] = sign_bits(d1); sf[n][3] = sign_bits(d3);
            }
            // dX^T += S^T W over the step's channels (y and the targets are dead here)
            const float* w0r = w + 2 * t * SW + 8 * kt0 + g;
#pragma unroll
            for (int nt = 0; nt < S::dkt; nt++)
#pragma unroll
                for (int n = 0; n < kNT; n++)
                    mma_tf32(dacc[nt], sf[n], __float_as_uint(w0r[8 * n * SW + 8 * nt]),
                             __float_as_uint(w0r[(8 * n + 1) * SW + 8 * nt]));
        }
    }

    if constexpr (LOSS) {
        // dL/dx: tile nt holds (pixel g / g + 8, input channel 8 nt + 2t / + 1); every element written once
#pragma unroll
        for (int nt = 0; nt < S::dkt; nt++) {
            const int c = 8 * (kt0 + nt) + 2 * t;
            if (c < Cin) {
                if (ina) a.dx[(size_t)c * N + pa] = a.grad_scale * dacc[nt][0];
                if (inb) a.dx[(size_t)c * N + pb] = a.grad_scale * dacc[nt][2];
            }
            if (c + 1 < Cin) {
                if (ina) a.dx[(size_t)(c + 1) * N + pa] = a.grad_scale * dacc[nt][1];
                if (inb) a.dx[(size_t)(c + 1) * N + pb] = a.grad_scale * dacc[nt][3];
            }
        }
        // per-CTA partial of sum |y - gt|, fixed reduction order
        __shared__ float red[kWarpsA];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        if (lane == 0) red[warp] = lsum;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = red[0];
            for (int i = 1; i < kWarpsA; i++) s += red[i];
            a.loss_part[blockIdx.x] = s;
        }
    }
}

// W -> TF32 [rows, Cp] zero-padded; b -> [rows] zero-padded (zeros without a bias)
__global__ void decoder_prep_kernel(int Cin, int Cout, int Cp, int rows, const float* __restrict__ W,
                                    const float* __restrict__ b, float* __restrict__ wt, float* __restrict__ bp) {
    const size_t n = (size_t)rows * Cp;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / Cp), c = (int)(i - (size_t)r * Cp);
        wt[i] = __uint_as_float(to_tf32(r < Cout && c < Cin ? W[(size_t)r * Cin + c] : 0.f));
        if (c == 0) bp[r] = b != nullptr && r < Cout ? b[r] : 0.f;
    }
}

// dW partial of one (128 output channels, 32 input channels, pixel range) tile: a warp owns 32 x 32 (2 x 4 mma tiles).
// K = pixels, 8 per k-step; slot t <-> pixel 2t and slot t + 4 <-> 2t + 1, so a thread's two x values are neighbours.
// The CTAs of input-channel tile 0 also count the signs of their rows (exact integers, for db).
__global__ void __launch_bounds__(kThreadsB) decoder_wgrad_kernel(int Cin, int Cout, int N, int N16, int Cp, int Cout_pad,
                                                                  int blk_per_split, const float* __restrict__ x,
                                                                  const uint32_t* __restrict__ bits,
                                                                  float* __restrict__ part_w, int* __restrict__ part_b) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int co0 = blockIdx.x * kCoutB + warp * 32, ci0 = blockIdx.y * kCinB, split = blockIdx.z;
    const int blk0 = split * blk_per_split, blk1 = min(N16, blk0 + blk_per_split);
    const bool count = blockIdx.y == 0 && t == 0;
    float acc[2][4][4];
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
        for (int nt = 0; nt < 4; nt++)
#pragma unroll
            for (int i = 0; i < 4; i++) acc[m][nt][i] = 0.f;
    int cnt[2][2] = {{0, 0}, {0, 0}};
    const float* xrow[4];
    bool xin[4];
#pragma unroll
    for (int nt = 0; nt < 4; nt++) {
        const int c = ci0 + 8 * nt + g;
        xin[nt] = c < Cin;
        xrow[nt] = x + (size_t)(xin[nt] ? c : 0) * N;
    }
    for (int blk = blk0; blk < blk1; blk++) {
        uint32_t wd[2][2];  // rows co0 + 16m + 8h + g
#pragma unroll
        for (int m = 0; m < 2; m++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int r = co0 + 16 * m + 8 * h + g;
                wd[m][h] = r < Cout ? __ldg(bits + (size_t)r * N16 + blk) : 0u;
                if (count) {
                    const uint32_t nz = wd[m][h] & 0xffffu, ng = wd[m][h] >> 16;
                    cnt[m][h] += __popc(nz) - 2 * __popc(ng);
                }
            }
#pragma unroll
        for (int hs = 0; hs < 2; hs++) {
            const int i = 8 * hs + 2 * t, p = blk * kPixWarp + i;
            uint32_t bf[4][2];
#pragma unroll
            for (int nt = 0; nt < 4; nt++) {
                bf[nt][0] = to_tf32(xin[nt] && p < N ? __ldg(xrow[nt] + p) : 0.f);
                bf[nt][1] = to_tf32(xin[nt] && p + 1 < N ? __ldg(xrow[nt] + p + 1) : 0.f);
            }
#pragma unroll
            for (int m = 0; m < 2; m++) {
                const uint32_t af[4] = {word_sign(wd[m][0], i), word_sign(wd[m][1], i), word_sign(wd[m][0], i + 1),
                                        word_sign(wd[m][1], i + 1)};
#pragma unroll
                for (int nt = 0; nt < 4; nt++) mma_tf32(acc[m][nt], af, bf[nt][0], bf[nt][1]);
            }
        }
    }
    // acc[m][nt]: (row co0 + 16m + g / + 8, column ci0 + 8nt + 2t / + 1); the partial is padded to [Cout_pad, Cp]
    float* pw = part_w + (size_t)split * Cout_pad * Cp;
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
        for (int nt = 0; nt < 4; nt++) {
            const int r = co0 + 16 * m + g, c = ci0 + 8 * nt + 2 * t;
            *reinterpret_cast<float2*>(pw + (size_t)r * Cp + c) = make_float2(acc[m][nt][0], acc[m][nt][1]);
            *reinterpret_cast<float2*>(pw + (size_t)(r + 8) * Cp + c) = make_float2(acc[m][nt][2], acc[m][nt][3]);
        }
    if (count) {
#pragma unroll
        for (int m = 0; m < 2; m++)
#pragma unroll
            for (int h = 0; h < 2; h++) part_b[(size_t)split * Cout_pad + co0 + 16 * m + 8 * h + g] = cnt[m][h];
    }
}

// dW[r, c] += gs * sum_split part_w;  db[r] += gs * sum_split part_b  (split order fixed)
__global__ void decoder_finish_kernel(int Cin, int Cout, int Cp, int Cout_pad, int splits, float gs,
                                      const float* __restrict__ part_w, const int* __restrict__ part_b,
                                      float* __restrict__ dW, float* __restrict__ db) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x, nw = (size_t)Cout * Cin;
    if (i < nw) {
        const int r = (int)(i / Cin), c = (int)(i - (size_t)r * Cin);
        float s = 0.f;
        for (int sp = 0; sp < splits; sp++) s += part_w[((size_t)sp * Cout_pad + r) * Cp + c];
        dW[i] += gs * s;
    } else if (db != nullptr && i < nw + Cout) {
        const int r = (int)(i - nw);
        int n = 0;
        for (int sp = 0; sp < splits; sp++) n += part_b[(size_t)sp * Cout_pad + r];
        db[r] += gs * (float)n;
    }
}

// One CTA sums the per-CTA loss partials in double, each thread a fixed strided subset, then a fixed tree.
__global__ void __launch_bounds__(kReduceThreads) decoder_loss_reduce_kernel(const float* __restrict__ part, size_t n,
                                                                              float* __restrict__ out) {
    __shared__ double r[kReduceThreads];
    double a = 0.0;
    for (size_t i = threadIdx.x; i < n; i += kReduceThreads) a += part[i];
    r[threadIdx.x] = a;
    __syncthreads();
    for (int s = kReduceThreads / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) r[threadIdx.x] += r[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = (float)r[0];
}

int kt_of(int Cin) { return Cin <= 32 ? 4 : Cin <= 64 ? 8 : Cin <= 128 ? 16 : 32; }

struct Plan {
    int KT, Cp, Cout_pad, N16, gridA, cin_tiles, splits, blk_per_split;
};

Plan make_plan(int Cin, int Cout, int N) {
    Plan p;
    p.KT = kt_of(Cin);
    p.Cp = 8 * p.KT;
    p.Cout_pad = (int)align_up(Cout, kCoutAlign);
    p.N16 = (N + kPixWarp - 1) / kPixWarp;
    const int pix_a = kPixWarp * kWarpsA / (p.KT <= 16 ? DecSmem<16>::share : DecSmem<32>::share);
    p.gridA = (N + pix_a - 1) / pix_a;
    p.cin_tiles = (Cin + kCinB - 1) / kCinB;
    const int tiles = p.Cout_pad / kCoutB * p.cin_tiles;
    const int want = std::max(1, std::min(p.N16, (kTargetCtasB + tiles - 1) / tiles));
    p.blk_per_split = (p.N16 + want - 1) / want;
    p.splits = (p.N16 + p.blk_per_split - 1) / p.blk_per_split;
    return p;
}

template <int KT, bool LOSS, typename T>
cudaError_t launch_a(const Plan& p, const DecArgs<T>& a, cudaStream_t s) {
    const size_t smem = DecSmem<KT>::bytes;
    cudaError_t e =
        cudaFuncSetAttribute(decoder_kernel<KT, LOSS, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    decoder_kernel<KT, LOSS, T><<<p.gridA, kThreadsA, smem, s>>>(a);
    return cudaGetLastError();
}

template <bool LOSS, typename T>
cudaError_t launch_a_kt(const Plan& p, const DecArgs<T>& a, cudaStream_t s) {
    switch (p.KT) {
        case 4: return launch_a<4, LOSS>(p, a, s);
        case 8: return launch_a<8, LOSS>(p, a, s);
        case 16: return launch_a<16, LOSS>(p, a, s);
        default: return launch_a<32, LOSS>(p, a, s);
    }
}

// stream-ordered scratch: W and b padded (both modes); signs, loss and split partials (loss mode)
struct Scratch {
    size_t off_wt = 0, off_bp, off_bits, off_loss, off_pw, off_pb, bytes;
    Scratch(const Plan& p, int Cout, bool loss) {
        size_t o = align_up((size_t)p.Cout_pad * p.Cp * 4, 256);
        off_bp = o;
        o = align_up(o + (size_t)p.Cout_pad * 4, 256);
        off_bits = off_loss = off_pw = off_pb = o;
        if (loss) {
            o = align_up(o + (size_t)Cout * p.N16 * 4, 256);
            off_loss = o;
            o = align_up(o + (size_t)p.gridA * 4, 256);
            off_pw = o;
            o = align_up(o + (size_t)p.splits * p.Cout_pad * p.Cp * 4, 256);
            off_pb = o;
            o += (size_t)p.splits * p.Cout_pad * 4;
        }
        bytes = o;
    }
};

template <typename T>
cudaError_t decoder_run(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x, const T* gt,
                        float grad_scale, T* y, float* loss_sum, float* dx, float* dW, float* db, cudaStream_t s) {
    if (!decoder_grid_ok(Cin, Cout, N)) return cudaErrorInvalidValue;
    const bool loss = gt != nullptr;
    const Plan p = make_plan(Cin, Cout, N);
    const Scratch sc(p, Cout, loss);
    char* ws = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&ws, sc.bytes, s);
    if (e != cudaSuccess) return e;
    DecArgs<T> a;
    a.Cin = Cin; a.Cout = Cout; a.N = N; a.N16 = p.N16;
    a.wt = reinterpret_cast<float*>(ws + sc.off_wt);
    a.bias = reinterpret_cast<float*>(ws + sc.off_bp);
    a.x = x; a.gt = gt; a.y = y; a.dx = dx;
    a.bits = reinterpret_cast<uint32_t*>(ws + sc.off_bits);
    a.loss_part = reinterpret_cast<float*>(ws + sc.off_loss);
    a.grad_scale = grad_scale;
    e = launch_decoder_prep(Cin, Cout, p.Cp, p.Cout_pad, weight, bias, const_cast<float*>(a.wt),
                            const_cast<float*>(a.bias), s);
    if (e == cudaSuccess) {
        e = loss ? launch_a_kt<true>(p, a, s) : launch_a_kt<false>(p, a, s);
        g_launches++;
    }
    if (e == cudaSuccess && loss) {
        float* pw = reinterpret_cast<float*>(ws + sc.off_pw);
        int* pb = reinterpret_cast<int*>(ws + sc.off_pb);
        decoder_wgrad_kernel<<<dim3(p.Cout_pad / kCoutB, p.cin_tiles, p.splits), kThreadsB, 0, s>>>(
            Cin, Cout, N, p.N16, p.Cp, p.Cout_pad, p.blk_per_split, x, a.bits, pw, pb);
        const size_t nfin = (size_t)Cout * Cin + Cout;
        decoder_finish_kernel<<<(unsigned)((nfin + 255) / 256), 256, 0, s>>>(Cin, Cout, p.Cp, p.Cout_pad, p.splits,
                                                                             grad_scale, pw, pb, dW, db);
        decoder_loss_reduce_kernel<<<1, kReduceThreads, 0, s>>>(a.loss_part, (size_t)p.gridA, loss_sum);
        g_launches += 3;
        e = cudaGetLastError();
    }
    cudaFreeAsync(ws, s);
    return e;
}

}  // namespace

cudaError_t launch_decoder_prep(int Cin, int Cout, int Cp, int rows, const float* weight, const float* bias, float* wt,
                                float* bp, cudaStream_t s) {
    const size_t n = (size_t)rows * Cp;
    decoder_prep_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, 1024), 256, 0, s>>>(Cin, Cout, Cp, rows, weight,
                                                                                        bias, wt, bp);
    g_launches++;
    return cudaGetLastError();
}

bool decoder_grid_ok(int Cin, int Cout, int N) {
    if (Cin < 1 || Cin > kDecoderMaxCin || Cout < 1 || Cout > kDecoderMaxCout || N < 1) return false;
    const Plan p = make_plan(Cin, Cout, N);
    return p.gridA <= 0x7fffffff && p.splits <= 65535 && p.cin_tiles <= 65535 &&
           (size_t)Cout * Cin + Cout <= (size_t)0x7fffffff * 256;
}

template <typename Y>
cudaError_t launch_decoder_forward(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x, Y* y,
                                   cudaStream_t s) {
    return decoder_run<Y>(Cin, Cout, N, weight, bias, x, nullptr, 0.f, y, nullptr, nullptr, nullptr, nullptr, s);
}
template cudaError_t launch_decoder_forward(int, int, int, const float*, const float*, const float*, float*, cudaStream_t);
template cudaError_t launch_decoder_forward(int, int, int, const float*, const float*, const float*, __half*, cudaStream_t);

template <typename GT>
cudaError_t launch_decoder_l1(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                              const GT* gt, float grad_scale, float* loss_sum, float* dx, float* dW, float* db,
                              cudaStream_t s) {
    return decoder_run<GT>(Cin, Cout, N, weight, bias, x, gt, grad_scale, nullptr, loss_sum, dx, dW, db, s);
}
template cudaError_t launch_decoder_l1(int, int, int, const float*, const float*, const float*, const float*, float, float*,
                                       float*, float*, float*, cudaStream_t);
template cudaError_t launch_decoder_l1(int, int, int, const float*, const float*, const float*, const __half*, float,
                                       float*, float*, float*, float*, cudaStream_t);

}  // namespace f3dgs
