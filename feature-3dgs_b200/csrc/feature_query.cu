// Text queries of a feature field: LSeg's open-vocabulary head on a rendered (or saved) feature map, and the CLIP-text
// selection of Gaussians in the reference's render_edit (gaussian_renderer/__init__.py:58-170).
// Shapes: x [C, N] (a map [C,H,W] as N = H W columns, or per-Gaussian features transposed), optional decoder W [D, C]
// and b [D] (the --speedup CNN_decoder), text [K, D].  For every column n:
//     y = W x_n + b (x_n without a decoder);  yh = y / max(||y||, 1e-12);  th_k = t_k / max(||t_k||, 1e-12)
//     l_k = scale <yh, th_k>;  label = argmax_k l_k (first maximal index; NaN counts as maximal, as in torch.argmax)
//     prob = sum over positive k of softmax_k(l)  (fp32, max-subtracted)
// In PyTorch this is a conv writing y [D, N], a normalize writing a copy of it, a matmul writing K x N logits and a
// softmax writing another K x N; here only the requested outputs reach memory:
//     prep   text rows normalised, rounded to TF32 and zero-padded to [Kp, Dp] (Kp = 8 * tiles, Dp a multiple of 32);
//            the positive mask padded to [Kp]; W and b through the decoder's own prep, to [Dp, Cp] and [Dp].
//     query  a warp owns 16 columns and walks D in steps of 32 channels (16 at C > 128, where X^T lives in shared
//            memory), W and the step's slice of the text double-buffered in shared memory by cp.async.  Per step:
//            Y^T[16, step] = X^T W^T + b exactly as decoder_kernel forms it (or x itself, loaded one step ahead),
//            ||y||^2 summed from the fp32 values, then  L^T[16, K] += Y^T Th^T  with Y^T rounded to TF32 straight from
//            the accumulator registers: the accumulator holds channels (2t, 2t + 1) where the A operand wants (t, t + 4),
//            so both operands use the slot permutation of feature_decoder.cu (slot t <-> 2t, slot t + 4 <-> 2t + 1).
//            The normalisation is applied once, l = scale * acc / max(||y||, 1e-12), after a quad shuffle completes
//            ||y||^2.  K > 128: the prompts go in equal chunks of at most 128 (16 n8 tiles = 64 accumulator registers),
//            y recomputed per chunk, with a running max, running softmax sums and a running argmax.
//     epilogue  argmax, softmax sums over all and over the positive prompts, from registers; the 4 lanes of a quad share
//            a column pair and reduce with shuffles in a fixed order.
// No float atomics and fixed summation orders: results are bitwise reproducible and do not depend on which outputs are
// requested.  With every prompt positive the two softmax sums are the same operations, so prob is exactly 1.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels.h"
#include "tf32_mma.cuh"

namespace f3dgs {
namespace {

constexpr int kWarps = 8, kThreads = 32 * kWarps;
constexpr int kCols = 16;      // columns per warp: the M = 16 rows of one mma tile
constexpr int kMaxTiles = 16;  // n8 prompt tiles per chunk: 128 prompts
constexpr int kDAlign = 32;    // Dp: a whole number of steps

template <int KT>  // decode in KT k8 steps (Cp = 8 KT >= C); KT = 0: no decoder
struct QSmem {
    static constexpr bool dec = KT > 0;
    static constexpr int Cp = 8 * KT, SW = Cp + 4;  // W rows padded by 4 floats, as in decoder_kernel
    static constexpr bool x_in_regs = KT <= 16;     // C > 128: X^T fragments in shared memory (128 registers would spill)
    static constexpr int step = x_in_regs ? 32 : 16;
    static constexpr int TS = step + 8;             // text rows padded by 8 floats: conflict-free 64-bit fragment loads
    static constexpr int xs_f4 = x_in_regs ? 0 : kWarps * KT * 32;
    static constexpr int w_floats = dec ? 2 * step * SW : 0;
    static constexpr int t_floats = 2 * kMaxTiles * 8 * TS;
    static constexpr size_t bytes = (size_t)xs_f4 * 16 + (size_t)(w_floats + t_floats) * 4;
};

template <typename T>  // element type of x: float or __half
struct QArgs {
    int C, D, K, N, Dp, tiles, chunks, chunk_tiles;
    const float* wt;      // [Dp, Cp] TF32, zero-padded          (decoder)
    const float* bias;    // [Dp], zero-padded                    (decoder)
    const T* x;           // [C, N]
    const float* text;    // [8 tiles, Dp] unit rows in TF32, zero-padded
    const uint8_t* pos;   // [8 tiles] 0/1
    float scale;
    int64_t* labels;      // [N]     or nullptr
    float* prob;          // [N]     or nullptr
    float* logits;        // [K, N]  or nullptr
};

// (vb, ib) replaces (va, ia) as the argmax: NaN counts as maximal (torch.argmax), ties go to the lower index.  A strict
// preference, so the two lanes of a shuffle pair pick the same winner.
__device__ __forceinline__ bool beats(float vb, int ib, float va, int ia) {
    if (va != va) return vb != vb && ib < ia;
    return vb != vb || vb > va || (vb == va && ib < ia);
}

template <int KT, typename T>
__global__ void __launch_bounds__(kThreads, 1) query_kernel(QArgs<T> a) {
    using S = QSmem<KT>;
    constexpr int Cp = S::Cp, SW = S::SW, TS = S::TS, kStep = S::step, kNT = kStep / 8;
    extern __shared__ float4 smem4[];
    float4* xs = smem4 + (threadIdx.x >> 5) * KT * 32;                  // this warp's [KT][32] fragments (C > 128)
    float* ws = reinterpret_cast<float*>(smem4 + S::xs_f4);             // [2][kStep][SW]        (decoder)
    float* ts = ws + S::w_floats;                                       // [2][8 kMaxTiles][TS]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int N = a.N, D = a.D;
    const int pa = (blockIdx.x * kWarps + warp) * kCols + g, pb = pa + 8;
    const bool ina = pa < N, inb = pb < N;
    const int steps = (D + kStep - 1) / kStep, stages = steps * a.chunks;

    // stage q = (chunk, step): W rows of the step and the text slice [chunk's prompts, step's channels]
    auto load_stage = [&](int q) {
        const int ch = q / steps, co = (q - ch * steps) * kStep;
        if constexpr (S::dec) {
            const float* src = a.wt + (size_t)co * Cp;
            float* dst = ws + (q & 1) * kStep * SW;
            for (int i = threadIdx.x; i < kStep * Cp / 4; i += kThreads) {
                const int r = i / (Cp / 4), c = (i - r * (Cp / 4)) * 4;
                cp_async16(dst + r * SW + c, src + (size_t)r * Cp + c);
            }
        }
        const int tile0 = ch * a.chunk_tiles, rows = 8 * min(a.chunk_tiles, a.tiles - tile0);
        const float* src = a.text + (size_t)tile0 * 8 * a.Dp + co;
        float* dst = ts + (q & 1) * kMaxTiles * 8 * TS;
        for (int i = threadIdx.x; i < rows * (kStep / 4); i += kThreads) {
            const int r = i / (kStep / 4), c = (i - r * (kStep / 4)) * 4;
            cp_async16(dst + r * TS + c, src + (size_t)r * a.Dp + c);
        }
        cp_async_commit();
    };
    load_stage(0);

    // decoder: X^T A-fragments (column, input channel), rounded to TF32, zero outside the map and past C
    uint32_t xr[S::dec && S::x_in_regs ? KT : 1][4];
    if constexpr (S::dec) {
#pragma unroll
        for (int kt = 0; kt < KT; kt++) {
            const int c0 = 8 * kt + t, c1 = c0 + 4;
            uint32_t f[4];
            f[0] = to_tf32(c0 < a.C && ina ? load_f32(a.x + (size_t)c0 * N + pa) : 0.f);
            f[1] = to_tf32(c0 < a.C && inb ? load_f32(a.x + (size_t)c0 * N + pb) : 0.f);
            f[2] = to_tf32(c1 < a.C && ina ? load_f32(a.x + (size_t)c1 * N + pa) : 0.f);
            f[3] = to_tf32(c1 < a.C && inb ? load_f32(a.x + (size_t)c1 * N + pb) : 0.f);
            if constexpr (S::x_in_regs) {
#pragma unroll
                for (int i = 0; i < 4; i++) xr[kt][i] = f[i];
            } else {
                xs[kt * 32 + lane] = make_float4(__uint_as_float(f[0]), __uint_as_float(f[1]), __uint_as_float(f[2]),
                                                 __uint_as_float(f[3]));
            }
        }
    }

    // no decoder: y of one step, (column g / g + 8, channel co + 8n + 2t / + 1), fetched one step ahead
    float xn[S::dec ? 1 : kNT][4];
    auto fetch_x = [&](int q) {
        const int co = (q % steps) * kStep;
#pragma unroll
        for (int n = 0; n < kNT; n++) {
            const int c = co + 8 * n + 2 * t;
            const bool va = c < D, vb = c + 1 < D;
            xn[n][0] = va && ina ? load_f32(a.x + (size_t)c * N + pa) : 0.f;
            xn[n][1] = vb && ina ? load_f32(a.x + (size_t)(c + 1) * N + pa) : 0.f;
            xn[n][2] = va && inb ? load_f32(a.x + (size_t)c * N + pb) : 0.f;
            xn[n][3] = vb && inb ? load_f32(a.x + (size_t)(c + 1) * N + pb) : 0.f;
        }
    };
    if constexpr (!S::dec) fetch_x(0);

    // running state of columns g (index 0) and g + 8 (index 1) over the chunks
    float best[2] = {-INFINITY, -INFINITY}, mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f}, psum[2] = {0.f, 0.f};
    int arg[2] = {0, 0};
    float acc[kMaxTiles][4];  // L^T tiles: (column g / g + 8, prompt k0 + 8j + 2t / + 1)
    float ss[2];              // this lane's share of ||y||^2

    for (int q = 0; q < stages; q++) {
        const int ch = q / steps, st = q - ch * steps, co = st * kStep;
        const int jn = min(a.chunk_tiles, a.tiles - ch * a.chunk_tiles);  // prompt tiles of this chunk
        if (st == 0) {
#pragma unroll
            for (int j = 0; j < kMaxTiles; j++)
#pragma unroll
                for (int i = 0; i < 4; i++) acc[j][i] = 0.f;
            ss[0] = ss[1] = 0.f;
        }
        cp_async_wait_all();
        __syncthreads();  // stage q has landed, and every warp is done with the buffer stage q + 1 overwrites
        if (q + 1 < stages) load_stage(q + 1);
        const float* w = ws + (q & 1) * kStep * SW;
        const float* tb = ts + (q & 1) * kMaxTiles * 8 * TS;

        // Y^T A-fragments of the second product: (column g / g + 8, slot t <-> channel 2t, slot t + 4 <-> 2t + 1)
        uint32_t af[kNT][4];
        float yv[kNT][4];
        if constexpr (S::dec) {
#pragma unroll
            for (int n = 0; n < kNT; n++) {
                const float b0 = __ldg(a.bias + co + 8 * n + 2 * t), b1 = __ldg(a.bias + co + 8 * n + 2 * t + 1);
                yv[n][0] = b0; yv[n][1] = b1; yv[n][2] = b0; yv[n][3] = b1;
            }
#pragma unroll
            for (int kt = 0; kt < KT; kt++) {
                uint32_t xf[4];
                if constexpr (S::x_in_regs) {
#pragma unroll
                    for (int i = 0; i < 4; i++) xf[i] = xr[kt][i];
                } else {
                    const float4 v = xs[kt * 32 + lane];
                    xf[0] = __float_as_uint(v.x); xf[1] = __float_as_uint(v.y);
                    xf[2] = __float_as_uint(v.z); xf[3] = __float_as_uint(v.w);
                }
#pragma unroll
                for (int n = 0; n < kNT; n++) {
                    const float* wr = w + (8 * n + g) * SW + 8 * kt + t;
                    mma_tf32(yv[n], xf, __float_as_uint(wr[0]), __float_as_uint(wr[4]));
                }
            }
        } else {
#pragma unroll
            for (int n = 0; n < kNT; n++)
#pragma unroll
                for (int i = 0; i < 4; i++) yv[n][i] = xn[n][i];
            if (q + 1 < stages) fetch_x(q + 1);
        }
#pragma unroll
        for (int n = 0; n < kNT; n++) {
            ss[0] += yv[n][0] * yv[n][0] + yv[n][1] * yv[n][1];
            ss[1] += yv[n][2] * yv[n][2] + yv[n][3] * yv[n][3];
            af[n][0] = to_tf32(yv[n][0]); af[n][1] = to_tf32(yv[n][2]);
            af[n][2] = to_tf32(yv[n][1]); af[n][3] = to_tf32(yv[n][3]);
        }

        // L^T += Y^T Th^T over the step's channels; b0 / b1 = Th[prompt 8j + g][channel co + 8n + 2t / + 1]
        const float* tr = tb + g * TS + 2 * t;
#pragma unroll
        for (int j = 0; j < kMaxTiles; j++) {
            if (j < jn) {
#pragma unroll
                for (int n = 0; n < kNT; n++) {
                    const float2 b = *reinterpret_cast<const float2*>(tr + 8 * j * TS + 8 * n);
                    mma_tf32(acc[j], af[n], __float_as_uint(b.x), __float_as_uint(b.y));
                }
            }
        }
        if (st != steps - 1) continue;

        // ---- chunk epilogue
        const int k0 = ch * a.chunk_tiles * 8;
        float f[2];
#pragma unroll
        for (int c = 0; c < 2; c++) {
            float s = ss[c];
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            f[c] = a.scale / fmaxf(sqrtf(s), 1e-12f);
        }
        const bool in[2] = {ina, inb};
        const int col[2] = {pa, pb};
        float cb[2] = {-INFINITY, -INFINITY};
        int ci[2] = {0x7fffffff, 0x7fffffff};
#pragma unroll
        for (int j = 0; j < kMaxTiles; j++) {
            if (j >= jn) continue;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int k = k0 + 8 * j + 2 * t + h;
                if (k >= a.K) continue;
#pragma unroll
                for (int c = 0; c < 2; c++) {
                    const float l = acc[j][2 * c + h] * f[c];
                    if (a.logits != nullptr && in[c]) a.logits[(size_t)k * N + col[c]] = l;
                    if (beats(l, k, cb[c], ci[c])) { cb[c] = l; ci[c] = k; }
                }
            }
        }
#pragma unroll
        for (int c = 0; c < 2; c++) {
#pragma unroll
            for (int o = 1; o < 4; o <<= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, cb[c], o);
                const int oi = __shfl_xor_sync(0xffffffffu, ci[c], o);
                if (beats(ob, oi, cb[c], ci[c])) { cb[c] = ob; ci[c] = oi; }
            }
            if (beats(cb[c], ci[c], best[c], arg[c])) { best[c] = cb[c]; arg[c] = ci[c]; }
        }
        if (a.prob == nullptr) continue;
#pragma unroll
        for (int c = 0; c < 2; c++) {
            const float m = fmaxf(mx[c], cb[c]), r = expf(mx[c] - m);
            float ls = 0.f, lp = 0.f;  // identical operations when every prompt is positive
#pragma unroll
            for (int j = 0; j < kMaxTiles; j++) {
                if (j >= jn) continue;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int k = k0 + 8 * j + 2 * t + h;
                    if (k >= a.K) continue;
                    const float e = expf(acc[j][2 * c + h] * f[c] - m);
                    ls += e;
                    lp += __ldg(a.pos + k) ? e : 0.f;
                }
            }
#pragma unroll
            for (int o = 1; o < 4; o <<= 1) {
                ls += __shfl_xor_sync(0xffffffffu, ls, o);
                lp += __shfl_xor_sync(0xffffffffu, lp, o);
            }
            sum[c] = sum[c] * r + ls;
            psum[c] = psum[c] * r + lp;
            mx[c] = m;
        }
    }

    if (t == 0) {
        if (ina) {
            if (a.labels != nullptr) a.labels[pa] = arg[0];
            if (a.prob != nullptr) a.prob[pa] = psum[0] / sum[0];
        }
        if (inb) {
            if (a.labels != nullptr) a.labels[pb] = arg[1];
            if (a.prob != nullptr) a.prob[pb] = psum[1] / sum[1];
        }
    }
}

// one warp per padded text row r: th_r = t_r / max(||t_r||, 1e-12) rounded to TF32 (zero past K and D); the positive
// mask as 0/1 (zero past K, and everywhere without a positive set)
__global__ void query_text_prep_kernel(int K, int D, int Dp, const float* __restrict__ text,
                                       const uint8_t* __restrict__ positive, float* __restrict__ th,
                                       uint8_t* __restrict__ mask) {
    const int r = blockIdx.x, lane = threadIdx.x;
    const float* row = text + (size_t)r * D;
    float ss = 0.f;
    if (r < K)
        for (int c = lane; c < D; c += 32) ss += row[c] * row[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);  // the same bits in every lane
    const float nrm = fmaxf(sqrtf(ss), 1e-12f);
    for (int c = lane; c < Dp; c += 32)
        th[(size_t)r * Dp + c] = __uint_as_float(to_tf32(r < K && c < D ? row[c] / nrm : 0.f));
    if (lane == 0) mask[r] = r < K && positive != nullptr && positive[r] != 0;
}

int kt_of(int C) { return C <= 32 ? 4 : C <= 64 ? 8 : C <= 128 ? 16 : 32; }
size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

template <int KT, typename T>
cudaError_t launch_query(const QArgs<T>& a, cudaStream_t s) {
    const size_t smem = QSmem<KT>::bytes;
    cudaError_t e = cudaFuncSetAttribute(query_kernel<KT, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const unsigned grid = (unsigned)(((size_t)a.N + kWarps * kCols - 1) / (kWarps * kCols));
    query_kernel<KT, T><<<grid, kThreads, smem, s>>>(a);
    g_launches++;
    return cudaGetLastError();
}

template <typename T>
cudaError_t query_run(int C, int D, int K, int N, const float* weight, const float* bias, const T* x, const float* text,
                      float scale, const uint8_t* positive, int64_t* labels, float* prob, float* logits,
                      cudaStream_t s) {
    if (N == 0) return cudaSuccess;
    const int KT = weight != nullptr ? kt_of(C) : 0, Cp = 8 * KT;
    QArgs<T> a;
    a.C = C; a.D = D; a.K = K; a.N = N;
    a.Dp = (int)round_up(D, kDAlign);
    a.tiles = (K + 7) / 8;
    a.chunks = (a.tiles + kMaxTiles - 1) / kMaxTiles;
    a.chunk_tiles = (a.tiles + a.chunks - 1) / a.chunks;  // equal chunks: K = 150 runs 2 x 80 prompts, not 128 + 128
    const int Kp = 8 * a.tiles;
    // stream-ordered scratch: W [Dp, Cp] and b [Dp] (decoder), text [Kp, Dp], mask [Kp]
    const size_t off_b = round_up((size_t)a.Dp * Cp * 4, 256);
    const size_t off_t = round_up(off_b + (weight != nullptr ? (size_t)a.Dp * 4 : 0), 256);
    const size_t off_m = round_up(off_t + (size_t)Kp * a.Dp * 4, 256);
    char* ws = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&ws, off_m + Kp, s);
    if (e != cudaSuccess) return e;
    a.wt = reinterpret_cast<float*>(ws);
    a.bias = reinterpret_cast<float*>(ws + off_b);
    a.x = x;
    a.text = reinterpret_cast<float*>(ws + off_t);
    a.pos = reinterpret_cast<uint8_t*>(ws + off_m);
    a.scale = scale;
    a.labels = labels; a.prob = prob; a.logits = logits;
    if (weight != nullptr)
        e = launch_decoder_prep(C, D, Cp, a.Dp, weight, bias, const_cast<float*>(a.wt), const_cast<float*>(a.bias), s);
    if (e == cudaSuccess) {
        query_text_prep_kernel<<<Kp, 32, 0, s>>>(K, D, a.Dp, text, positive, const_cast<float*>(a.text),
                                                 const_cast<uint8_t*>(a.pos));
        g_launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        switch (KT) {
            case 0: e = launch_query<0>(a, s); break;
            case 4: e = launch_query<4>(a, s); break;
            case 8: e = launch_query<8>(a, s); break;
            case 16: e = launch_query<16>(a, s); break;
            default: e = launch_query<32>(a, s); break;
        }
    }
    cudaFreeAsync(ws, s);
    return e;
}

}  // namespace

cudaError_t launch_feature_query(int C, int D, int K, int N, const float* weight, const float* bias, const float* x,
                                 const float* text, float logit_scale, const uint8_t* positive, int64_t* labels,
                                 float* prob, float* logits, cudaStream_t s) {
    return query_run<float>(C, D, K, N, weight, bias, x, text, logit_scale, positive, labels, prob, logits, s);
}

cudaError_t launch_feature_query(int C, int D, int K, int N, const float* weight, const float* bias, const __half* x,
                                 const float* text, float logit_scale, const uint8_t* positive, int64_t* labels,
                                 float* prob, float* logits, cudaStream_t s) {
    return query_run<__half>(C, D, K, N, weight, bias, x, text, logit_scale, positive, labels, prob, logits, s);
}

}  // namespace f3dgs
