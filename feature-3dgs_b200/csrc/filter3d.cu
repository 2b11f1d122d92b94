// Mip-Splatting's 3D smoothing filter (Yu et al., CVPR 2024; the official scene/gaussian_model.py compute_3D_filter,
// get_scaling_with_3D_filter, get_opacity_with_3D_filter, reset_opacity).  See include/f3dgs_b200.h: f3dgs_filter3d_*.
//
// compute  two kernels.  filter3d_distance_kernel: one thread per Gaussian, the cameras staged through shared memory in
//          chunks of kCamChunk; per Gaussian the min depth over the cameras that see it (or -1 if none), and per block
//          the seen count (one integer atomicAdd) and the max seen depth (one integer atomicMax on the float bits: all
//          depths are > 0.2, so their bit patterns order as the floats do).  filter3d_finish_kernel: unseen rows take
//          that max, and every row is scaled by sqrt(0.2) / focal with focal the max fx over the cameras.  min, max and
//          integer counts are exact, so the result is bitwise deterministic and independent of the camera order.
// apply    elementwise (o, s, f) -> (o * coef, sqrt(s^2 + f^2)), coef = sqrt(det1 / det2), in the official torch
//          formula's float32 operations (no contraction: nvcc's default -fmad=true would fuse s^2 + f^2).
// backward elementwise, in place over the gradient buffers allowed.
// reset    the official filtered reset_opacity from the raw parameters, in place.
#include <cmath>

#include "kernels.h"

namespace f3dgs {

namespace {

constexpr int kThreads = 256;
constexpr int kCamChunk = 128;  // cameras per shared-memory stage (20 floats each: 10 KiB)
constexpr int kCamFloats = 20;  // vm rows 0-3 x cols 0-2 (12), fx, fy, W / 2, H / 2, x range, y range

// The camera terms of the official per-camera loop, in float32 as torch evaluates them: the screen margins are Python
// doubles (-0.15 * W, W * 1.15) rounded once to float for the comparison.
__device__ void stage_camera(const float* __restrict__ vm, const float* __restrict__ intr, float* __restrict__ out) {
    for (int r = 0; r < 4; r++)
        for (int c = 0; c < 3; c++) out[3 * r + c] = vm[4 * r + c];
    const float W = intr[2], H = intr[3];
    out[12] = intr[0];
    out[13] = intr[1];
    out[14] = (float)((double)W / 2.0);
    out[15] = (float)((double)H / 2.0);
    out[16] = (float)(-0.15 * (double)W);
    out[17] = (float)((double)W * 1.15);
    out[18] = (float)(-0.15 * (double)H);
    out[19] = (float)(1.15 * (double)H);
}

__global__ void __launch_bounds__(kThreads) filter3d_distance_kernel(int P, int V, const float* __restrict__ means3D,
                                                                     const float* __restrict__ viewmatrices,
                                                                     const float* __restrict__ intrinsics,
                                                                     float* __restrict__ filter, int* __restrict__ n_seen,
                                                                     unsigned* __restrict__ max_bits) {
    __shared__ float cam[kCamChunk * kCamFloats];
    __shared__ int s_seen;
    __shared__ unsigned s_max;
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (threadIdx.x == 0) {
        s_seen = 0;
        s_max = 0u;
    }
    float x0 = 0.f, x1 = 0.f, x2 = 0.f;
    if (i < P) {
        x0 = means3D[3 * i];
        x1 = means3D[3 * i + 1];
        x2 = means3D[3 * i + 2];
    }
    float dist = 100000.0f;
    bool seen = false;
    for (int c0 = 0; c0 < V; c0 += kCamChunk) {
        const int n = min(kCamChunk, V - c0);
        __syncthreads();  // the previous chunk is consumed
        for (int c = threadIdx.x; c < n; c += kThreads)
            stage_camera(viewmatrices + 16 * (size_t)(c0 + c), intrinsics + 4 * (size_t)(c0 + c), cam + kCamFloats * c);
        __syncthreads();
        if (i >= P) continue;
        for (int c = 0; c < n; c++) {
            const float* k = cam + kCamFloats * c;
            // xyz @ vm[:3,:3] + vm[3,:3], column j: the product in one fixed fma order, then the translation
            const float xc = __fadd_rn(fmar(x2, k[6], fmar(x1, k[3], mulr(x0, k[0]))), k[9]);
            const float yc = __fadd_rn(fmar(x2, k[7], fmar(x1, k[4], mulr(x0, k[1]))), k[10]);
            const float z = __fadd_rn(fmar(x2, k[8], fmar(x1, k[5], mulr(x0, k[2]))), k[11]);
            const float zc = fmaxf(z, 0.001f);
            const float px = addr(mulr(divr(xc, zc), k[12]), k[14]);
            const float py = addr(mulr(divr(yc, zc), k[13]), k[15]);
            const bool valid = z > 0.2f && px >= k[16] && px <= k[17] && py >= k[18] && py <= k[19];
            if (valid) {
                dist = fminf(dist, zc);
                seen = true;
            }
        }
    }
    if (i < P) filter[i] = seen ? dist : -1.0f;
    // every thread of the block is here (rows past P are unseen): the warp's count and max, then one shared atomic each
    const unsigned mask = __ballot_sync(0xffffffffu, seen);
    unsigned m = seen ? __float_as_uint(dist) : 0u;
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && mask) {
        atomicAdd(&s_seen, __popc(mask));
        atomicMax(&s_max, m);
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_seen > 0) {
        atomicAdd(n_seen, s_seen);
        atomicMax(max_bits, s_max);
    }
}

__global__ void __launch_bounds__(kThreads) filter3d_finish_kernel(int P, int V, const float* __restrict__ intrinsics,
                                                                   const unsigned* __restrict__ max_bits,
                                                                   float* __restrict__ filter) {
    __shared__ float s_focal[kThreads / 32];
    float f = 0.0f;
    for (int c = threadIdx.x; c < V; c += kThreads) f = fmaxf(f, intrinsics[4 * (size_t)c]);
    for (int o = 16; o > 0; o >>= 1) f = fmaxf(f, __shfl_xor_sync(0xffffffffu, f, o));
    if ((threadIdx.x & 31) == 0) s_focal[threadIdx.x >> 5] = f;
    __syncthreads();
    float focal = s_focal[0];
    for (int w = 1; w < kThreads / 32; w++) focal = fmaxf(focal, s_focal[w]);
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= P) return;
    const float d = filter[i];
    const float dist = d < 0.0f ? __uint_as_float(*max_bits) : d;
    // torch: distance / focal_length multiplies by the float reciprocal of the Python scalar; * (0.2 ** 0.5) rounds the
    // scalar to float
    filter[i] = mulr(mulr(dist, divr(1.0f, focal)), (float)0.4472135954999579);
}

// The official formula's per-Gaussian terms: s_k^2, f^2, s_f_k = sqrt(s_k^2 + f^2) and coef = sqrt(det1 / det2).  The
// determinants are multiplied in torch's .prod(dim=1) order on CUDA: a [P,3] row is reduced by two lanes, lane 0
// holding elements 0 and 2 and lane 1 element 1, so det = (a0 a2) a1.
struct Filtered {
    float s2[3], sf[3], f2, coef;
};

__device__ __forceinline__ Filtered filtered(const float s[3], float f) {
    Filtered r;
    r.f2 = mulr(f, f);
    float a[3];
    for (int k = 0; k < 3; k++) {
        r.s2[k] = mulr(s[k], s[k]);
        a[k] = addr(r.s2[k], r.f2);
        r.sf[k] = sqrtr(a[k]);
    }
    const float det1 = mulr(mulr(r.s2[0], r.s2[2]), r.s2[1]);
    const float det2 = mulr(mulr(a[0], a[2]), a[1]);
    r.coef = sqrtr(divr(det1, det2));
    return r;
}

__global__ void __launch_bounds__(kThreads) filter3d_apply_kernel(int P, const float* __restrict__ opacity,
                                                                  const float* __restrict__ scales,
                                                                  const float* __restrict__ filter,
                                                                  float* __restrict__ opacity_out,
                                                                  float* __restrict__ scales_out) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= P) return;
    const float s[3] = {scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]};
    const Filtered r = filtered(s, filter[i]);
    opacity_out[i] = mulr(opacity[i], r.coef);
    for (int k = 0; k < 3; k++) scales_out[3 * i + k] = r.sf[k];
}

// No __restrict__ on the gradients: dL_dopacity may be dL_dopacity_f and dL_dscales dL_dscales_f (every element is read
// before its own thread writes it).
__global__ void __launch_bounds__(kThreads) filter3d_apply_backward_kernel(int P, const float* __restrict__ opacity,
                                                                           const float* __restrict__ scales,
                                                                           const float* __restrict__ filter,
                                                                           const float* g_of, const float* g_sf,
                                                                           float* g_o, float* g_s) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= P) return;
    const float s[3] = {scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]};
    const Filtered r = filtered(s, filter[i]);
    const float go = g_of[i];
    const float gs[3] = {g_sf[3 * i], g_sf[3 * i + 1], g_sf[3 * i + 2]};
    const float of = opacity[i] * r.coef;
    g_o[i] = go * r.coef;
    for (int k = 0; k < 3; k++) {
        // d s_f / d s = s / s_f;  d o_f / d s = o_f f^2 / (s s_f^2), written as (o_f / s) (f^2 / s_f^2) so that no
        // intermediate leaves the range of its factors; 0 where o_f == 0 (an underflowed det1, or s == 0)
        float t = gs[k] * (s[k] / r.sf[k]);
        if (of != 0.0f) t += go * (of / s[k]) * (r.f2 / (r.sf[k] * r.sf[k]));
        g_s[3 * i + k] = t;
    }
}

__global__ void __launch_bounds__(kThreads) filter3d_reset_kernel(int P, float* __restrict__ raw_opacity,
                                                                  const float* __restrict__ raw_scaling,
                                                                  const float* __restrict__ filter,
                                                                  float* __restrict__ m, float* __restrict__ v,
                                                                  float ceiling) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= P) return;
    const float o = 1.0f / (1.0f + expf(-raw_opacity[i]));  // torch.sigmoid
    const float s[3] = {expf(raw_scaling[3 * i]), expf(raw_scaling[3 * i + 1]), expf(raw_scaling[3 * i + 2])};
    const Filtered r = filtered(s, filter[i]);
    const float of = mulr(o, r.coef);
    float x;
    if (r.coef != 0.0f) {
        x = (of != of) ? of : fminf(of, ceiling);  // torch.minimum: NaN propagates
        x = divr(x, r.coef);
    } else {
        x = (o != o) ? o : fminf(o, ceiling);  // the official 0 / 0: the unfiltered reset instead
    }
    raw_opacity[i] = logf(divr(x, subr(1.0f, x)));  // inverse_sigmoid
    m[i] = 0.0f;
    v[i] = 0.0f;
}

}  // namespace

cudaError_t launch_filter3d_compute(int P, int V, const float* means3D, const float* viewmatrices,
                                    const float* intrinsics, float* filter, int32_t* n_seen, char* scratch,
                                    cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    unsigned* max_bits = reinterpret_cast<unsigned*>(scratch);
    cudaError_t e;
    if ((e = cudaMemsetAsync(n_seen, 0, sizeof(int32_t), s)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(max_bits, 0, sizeof(unsigned), s)) != cudaSuccess) return e;
    filter3d_distance_kernel<<<blocks_for(P), kThreads, 0, s>>>(P, V, means3D, viewmatrices, intrinsics, filter,
                                                                 n_seen, max_bits);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    filter3d_finish_kernel<<<blocks_for(P), kThreads, 0, s>>>(P, V, intrinsics, max_bits, filter);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_filter3d_apply(int P, const float* opacity, const float* scales, const float* filter,
                                  float* opacity_out, float* scales_out, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    filter3d_apply_kernel<<<blocks_for(P), kThreads, 0, s>>>(P, opacity, scales, filter, opacity_out, scales_out);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_filter3d_apply_backward(int P, const float* opacity, const float* scales, const float* filter,
                                           const float* dL_dopacity_f, const float* dL_dscales_f, float* dL_dopacity,
                                           float* dL_dscales, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    filter3d_apply_backward_kernel<<<blocks_for(P), kThreads, 0, s>>>(P, opacity, scales, filter, dL_dopacity_f,
                                                                       dL_dscales_f, dL_dopacity, dL_dscales);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_reset_opacity_filter3d(int P, float* raw_opacity, const float* raw_scaling, const float* filter,
                                          float* exp_avg, float* exp_avg_sq, float ceiling, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    filter3d_reset_kernel<<<blocks_for(P), kThreads, 0, s>>>(P, raw_opacity, raw_scaling, filter, exp_avg, exp_avg_sq,
                                                              ceiling);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace f3dgs
