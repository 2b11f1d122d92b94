// Per-Gaussian terms over the k-NN graph of knn.cu (include/f3dgs_b200.h: f3dgs_feature_tv_accum, f3dgs_feature_fill).
//
// Total variation of the feature field over the graph's valid edges E (Gaussian Grouping's 3-D neighbour term, in L1):
//   L = weight / (|E| C) * sum_{(i,j) in E} sum_c |f_ic - f_jc|
//   dL/df_i = s * n_i,   s = float(weight / (|E| C)),   n_i = sum_{j in N(i)} sign(f_i - f_j) - sum_{i' in R(i)} sign(f_i' - f_i)
// tv_kernel gives one row to a warp, lanes over C (float4 when the rows allow it).  The row's forward neighbours come from
// idx, its sources from the reverse lists (CSR offsets / sources), so n_i is an integer count per channel, formed
// without atomics, and grad_i += float(n_i) * s is one product and one add, both rounded to nearest: the gradient is
// defined bitwise.  The loss is summed in double per row (lanes over C, then a fixed shuffle tree), stored by row, and
// reduced over rows in a fixed order by sum_kernel, so neither depends on the walk order.  Rows are walked in the graph's
// Morton order when given, so the neighbour rows a warp reads were read by nearby warps and are resident in L2.
//
// Neighbour fill (fill_kernel): a row with weight <= min_weight becomes sum_j w_j f_j / sum_j w_j over its neighbours
// with w_j > min_weight, both sums in double in neighbour order, the quotient rounded once to float; every other row,
// and a row without such a neighbour, is copied bitwise.
#include <algorithm>
#include <cmath>
#include <initializer_list>

#include "kernels.h"

namespace f3dgs {

namespace {

constexpr int kRowsPerCta = 8;  // one warp per row
constexpr int kSumThreads = 256;
constexpr int kSumBlocks = 1024;

template <int V>
struct Vec;
template <>
struct Vec<1> {
    float v[1];
    __device__ __forceinline__ void load(const float* p) { v[0] = *p; }
    __device__ __forceinline__ void store(float* p) const { *p = v[0]; }
};
template <>
struct Vec<4> {
    float v[4];
    __device__ __forceinline__ void load(const float* p) {
        const float4 t = *reinterpret_cast<const float4*>(p);
        v[0] = t.x;
        v[1] = t.y;
        v[2] = t.z;
        v[3] = t.w;
    }
    __device__ __forceinline__ void store(float* p) const {
        *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    }
};

__device__ __forceinline__ int sgn(float a, float b) { return (a > b) - (a < b); }

template <int V>
__global__ void __launch_bounds__(32 * kRowsPerCta) tv_kernel(int P, int k, int C, const float* __restrict__ f,
                                                              const int32_t* __restrict__ idx,
                                                              const int32_t* __restrict__ offsets,
                                                              const int32_t* __restrict__ sources,
                                                              const int32_t* __restrict__ order, float s,
                                                              float* __restrict__ grad, double* __restrict__ row_loss) {
    const int lane = threadIdx.x & 31;
    const long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    if (w >= P) return;  // warp-uniform
    const int i = order ? order[w] : (int)w;
    const int32_t nb = lane < k ? idx[(size_t)i * k + lane] : -1;
    const int r0 = offsets[i], r1 = offsets[i + 1];
    const float* fi = f + (size_t)i * C;
    float* gi = grad + (size_t)i * C;
    double loss = 0.0;
    for (int c0 = 0; c0 < C; c0 += 32 * V) {
        const int c = c0 + lane * V;
        const bool on = c < C;
        Vec<V> own, other;
        int n[V];
#pragma unroll
        for (int v = 0; v < V; v++) n[v] = 0;
        if (on) own.load(fi + c);
        for (int j = 0; j < k; j++) {
            const int32_t nj = __shfl_sync(0xffffffffu, nb, j);
            if (nj < 0 || nj >= P || !on) continue;  // -1: no neighbour
            other.load(f + (size_t)nj * C + c);
#pragma unroll
            for (int v = 0; v < V; v++) {
                n[v] += sgn(own.v[v], other.v[v]);
                loss += fabs((double)own.v[v] - (double)other.v[v]);
            }
        }
        if (!on) continue;
        for (int r = r0; r < r1; r++) {
            other.load(f + (size_t)sources[r] * C + c);
#pragma unroll
            for (int v = 0; v < V; v++) n[v] -= sgn(other.v[v], own.v[v]);
        }
        Vec<V> g;
        g.load(gi + c);
#pragma unroll
        for (int v = 0; v < V; v++) g.v[v] = __fadd_rn(g.v[v], __fmul_rn((float)n[v], s));
        g.store(gi + c);
    }
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    if (lane == 0) row_loss[i] = loss;
}

// out[b] = scale * the sum of in[b * chunk, min((b + 1) * chunk, n)), in a fixed order
__global__ void __launch_bounds__(kSumThreads) sum_kernel(long long n, long long chunk, const double* __restrict__ in,
                                                          double scale, double* __restrict__ out) {
    __shared__ double part[kSumThreads];
    const long long b0 = blockIdx.x * chunk, b1 = min(n, b0 + chunk);
    double acc = 0.0;
    for (long long r = b0 + threadIdx.x; r < b1; r += kSumThreads) acc += in[r];
    part[threadIdx.x] = acc;
    __syncthreads();
    for (int h = kSumThreads / 2; h > 0; h >>= 1) {
        if ((int)threadIdx.x < h) part[threadIdx.x] += part[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[blockIdx.x] = part[0] * scale;
}

template <int V>
__global__ void __launch_bounds__(32 * kRowsPerCta) fill_kernel(int P, int k, int C, const float* __restrict__ f,
                                                                const float* __restrict__ weight,
                                                                const int32_t* __restrict__ idx, float min_weight,
                                                                float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    if (w >= P) return;  // warp-uniform
    const int i = (int)w;
    const int32_t nb = lane < k ? idx[(size_t)i * k + lane] : -1;
    const float wn = nb >= 0 && nb < P ? weight[nb] : 0.f;
    const unsigned use = __ballot_sync(0xffffffffu, nb >= 0 && nb < P && wn > min_weight);
    const float* fi = f + (size_t)i * C;
    float* oi = out + (size_t)i * C;
    if (!(weight[i] <= min_weight) || use == 0) {
        for (int c = lane * V; c < C; c += 32 * V) {
            Vec<V> t;
            t.load(fi + c);
            t.store(oi + c);
        }
        return;
    }
    double wsum = 0.0;
    for (unsigned m = use; m; m &= m - 1) wsum += (double)__shfl_sync(0xffffffffu, wn, __ffs(m) - 1);
    for (int c0 = 0; c0 < C; c0 += 32 * V) {
        const int c = c0 + lane * V;
        const bool on = c < C;
        double acc[V];
#pragma unroll
        for (int v = 0; v < V; v++) acc[v] = 0.0;
        for (unsigned m = use; m; m &= m - 1) {
            const int j = __ffs(m) - 1;
            const int32_t nj = __shfl_sync(0xffffffffu, nb, j);
            const double wj = (double)__shfl_sync(0xffffffffu, wn, j);
            if (!on) continue;
            Vec<V> t;
            t.load(f + (size_t)nj * C + c);
#pragma unroll
            for (int v = 0; v < V; v++) acc[v] += wj * (double)t.v[v];
        }
        if (!on) continue;
        Vec<V> r;
#pragma unroll
        for (int v = 0; v < V; v++) r.v[v] = (float)(acc[v] / wsum);
        r.store(oi + c);
    }
}

// 128-bit rows: C a multiple of 4 and every base 16-byte aligned
bool vec4_ok(int C, std::initializer_list<const void*> ptrs) {
    if (C % 4) return false;
    for (const void* p : ptrs)
        if ((uintptr_t)p % 16) return false;
    return true;
}

unsigned row_blocks(int P) { return (unsigned)(((long long)P + kRowsPerCta - 1) / kRowsPerCta); }

}  // namespace

cudaError_t launch_feature_tv_accum(int P, int k, int C, const float* features, const int32_t* idx,
                                    const int32_t* offsets, const int32_t* sources, const int32_t* order, double weight,
                                    long long n_edges, float* grad, double* loss, cudaStream_t s) {
    if (P <= 0) return cudaSuccess;
    if (n_edges == 0) return cudaMemsetAsync(loss, 0, sizeof(double), s);
    const double scale = weight / ((double)n_edges * (double)C);
    const unsigned G = (unsigned)std::min<long long>(kSumBlocks, ((long long)P + 4095) / 4096);
    const long long chunk = ((long long)P + G - 1) / G;
    double* ws = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&ws, ((size_t)P + G) * sizeof(double), s);
    if (e != cudaSuccess) return e;
    if (vec4_ok(C, {features, grad}))
        tv_kernel<4><<<row_blocks(P), 32 * kRowsPerCta, 0, s>>>(P, k, C, features, idx, offsets, sources, order,
                                                                (float)scale, grad, ws);
    else
        tv_kernel<1><<<row_blocks(P), 32 * kRowsPerCta, 0, s>>>(P, k, C, features, idx, offsets, sources, order,
                                                                (float)scale, grad, ws);
    sum_kernel<<<G, kSumThreads, 0, s>>>(P, chunk, ws, 1.0, ws + P);
    sum_kernel<<<1, kSumThreads, 0, s>>>(G, G, ws + P, scale, loss);
    g_launches += 3;
    e = cudaGetLastError();
    const cudaError_t f = cudaFreeAsync(ws, s);
    return e != cudaSuccess ? e : f;
}

cudaError_t launch_feature_fill(int P, int k, int C, const float* features, const float* weight, const int32_t* idx,
                                float min_weight, float* out, cudaStream_t s) {
    if (P <= 0) return cudaSuccess;
    if (vec4_ok(C, {features, out}))
        fill_kernel<4><<<row_blocks(P), 32 * kRowsPerCta, 0, s>>>(P, k, C, features, weight, idx, min_weight, out);
    else
        fill_kernel<1><<<row_blocks(P), 32 * kRowsPerCta, 0, s>>>(P, k, C, features, weight, idx, min_weight, out);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace f3dgs
