// Photometric image loss of the reference training step: L1 + D-SSIM with its gradient w.r.t. the rendered image.
// Reference: train.py (loss = (1 - lambda_dssim) * l1_loss(image, gt) + lambda_dssim * (1 - ssim(image, gt)))
//            utils/loss_utils.py  l1_loss, ssim(window_size=11, size_average=True)
// The reference's ssim is five depthwise 11x11 F.conv2d calls (zero padding 5, one Gaussian window per channel, sigma 1.5)
// plus a dozen elementwise kernels, and autograd runs their transposes.  Here ONE kernel per call computes sum |x - y|,
// sum S and, optionally, dL/dx = w_l1 * sign(x - y) + w_ssim * d(sum S)/dx, where with mx = blur(x), mxx = blur(x^2) ...
//     dS/dmx  = S (2my/A1 - 2my/A2 - 2mx/B1 + 2mx/B2)   dS/dmxx = -S/B2   dS/dmxy = 2S/A2
//     d(sum S)/dx = blur(dS/dmx) + 2x blur(dS/dmxx) + y blur(dS/dmxy)
// (the window is symmetric and zero-padded, so blur is its own transpose).  A CTA owns a kTX x kTY tile of one plane and
// recomputes its halo instead of exchanging it through global scratch:
//     stage x, y on the tile + 10 px (zero outside the image, which is the zero padding of every blurred map)
//  -> horizontal blur of the five products x, y, x^2, y^2, xy on the tile + 5 px columns
//  -> vertical blur to the five moments on the tile + 5 px, S and the three dS/dm maps (zero outside the image)
//  -> horizontal then vertical blur of the three maps down to the tile, combined with x, y and the L1 sign.
// DRAM traffic is one read of x and y and one write of the gradient.  Every gradient element is written exactly once
// (no zero fill, no atomics), and both sums are per-CTA partials reduced in a fixed order, so the results are bitwise
// reproducible run to run.
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>

#include "kernels.h"

namespace f3dgs {
namespace {

constexpr int kTX = 32, kTY = 16;  // output tile
constexpr int kR = 5;              // window radius (11 taps)
constexpr int kTaps = 2 * kR + 1;
constexpr int kThreads = 256;
constexpr int kSX = kTX + 4 * kR, kSY = kTY + 4 * kR;  // staged x, y: tile + 10 px

struct Window {
    float w[kTaps];
};

// Rows / columns of each stage; the value-only kernel needs the moments on the tile alone (halo 0 instead of kR).
template <bool GRAD>
struct Dims {
    static constexpr int halo = GRAD ? kR : 0;
    static constexpr int mcols = kTX + 2 * halo;    // columns of the horizontal moment pass and of the moments
    static constexpr int mrows = kTY + 2 * halo;    // rows of the moments
    static constexpr int hrows = mrows + 2 * kR;    // rows of the horizontal moment pass
    static constexpr int off = kR - halo;           // first staged row / column the horizontal pass reads from
    static constexpr int smem_floats = 2 * kSY * kSX + 5 * hrows * mcols + (GRAD ? 3 * mrows * mcols : 0);
};

constexpr float kC1 = 0.01f * 0.01f, kC2 = 0.03f * 0.03f;

template <bool GRAD>
__global__ void __launch_bounds__(kThreads, 3)
image_loss_kernel(int H, int W, Window win, const float* __restrict__ image, const float* __restrict__ gt, float w_l1,
                  float w_ssim, float2* __restrict__ partial, float* __restrict__ dL_dimage) {
    using D = Dims<GRAD>;
    extern __shared__ float smem[];
    float* sx = smem;                        // [kSY][kSX]
    float* sy = sx + kSY * kSX;              // [kSY][kSX]
    float* hm = sy + kSY * kSX;              // [5][hrows][mcols]  horizontal blur of x, y, x^2, y^2, xy
    float* dm = hm + 5 * D::hrows * D::mcols;  // [3][mrows][mcols]  dS/dmx, dS/dmxx, dS/dmxy (GRAD only)
    float* hd = hm;                          // [3][mrows][kTX]    horizontal blur of dm (reuses hm)
    // the SSIM map on the tile, summed in the same order as the L1 term so that both modes give the same sums
    __shared__ float s_map[kTY * kTX];

    const int tid = threadIdx.x;
    const int tx0 = blockIdx.x * kTX, ty0 = blockIdx.y * kTY;
    const size_t plane = (size_t)blockIdx.z * H * W;
    const float* xp = image + plane;
    const float* yp = gt + plane;

    // ---- stage x, y with a 2 * kR halo, zero outside the image
    {
        constexpr int kPer = (kSY * kSX + kThreads - 1) / kThreads;  // all loads of a thread in flight at once
        float lx[kPer], ly[kPer];
#pragma unroll
        for (int k = 0; k < kPer; k++) {
            const int i = tid + k * kThreads;
            const int r = i / kSX, c = i - r * kSX;
            const int gy = ty0 - 2 * kR + r, gx = tx0 - 2 * kR + c;
            const bool in = i < kSY * kSX && gy >= 0 && gy < H && gx >= 0 && gx < W;
            const size_t o = (size_t)gy * W + gx;
            lx[k] = in ? __ldg(xp + o) : 0.f;
            ly[k] = in ? __ldg(yp + o) : 0.f;
        }
#pragma unroll
        for (int k = 0; k < kPer; k++) {
            const int i = tid + k * kThreads;
            if (i < kSY * kSX) {
                sx[i] = lx[k];
                sy[i] = ly[k];
            }
        }
    }
    __syncthreads();

    // ---- horizontal blur of the five products; a thread owns a run of kRunH consecutive output columns of one row
    {
        constexpr int kRunH = GRAD ? 6 : 4;
        constexpr int runs = (D::mcols + kRunH - 1) / kRunH;
        static_assert(D::mcols % kRunH == 0, "runs tile the columns");
        for (int it = tid; it < D::hrows * runs; it += kThreads) {
            const int r = it / runs, c0 = (it - r * runs) * kRunH;
            const float* px = sx + (r + D::off) * kSX + c0 + D::off;
            const float* py = sy + (r + D::off) * kSX + c0 + D::off;
            float vx[kRunH + 2 * kR], vy[kRunH + 2 * kR];
#pragma unroll
            for (int k = 0; k < kRunH + 2 * kR; k++) {
                vx[k] = px[k];
                vy[k] = py[k];
            }
            float acc[5][kRunH];
#pragma unroll
            for (int j = 0; j < kRunH; j++) {
#pragma unroll
                for (int m = 0; m < 5; m++) acc[m][j] = 0.f;
#pragma unroll
                for (int t = 0; t < kTaps; t++) {
                    const float a = vx[j + t], b = vy[j + t], w = win.w[t];
                    acc[0][j] = fmaf(w, a, acc[0][j]);
                    acc[1][j] = fmaf(w, b, acc[1][j]);
                    acc[2][j] = fmaf(w, a * a, acc[2][j]);
                    acc[3][j] = fmaf(w, b * b, acc[3][j]);
                    acc[4][j] = fmaf(w, a * b, acc[4][j]);
                }
            }
#pragma unroll
            for (int m = 0; m < 5; m++)
#pragma unroll
                for (int j = 0; j < kRunH; j++) hm[(m * D::hrows + r) * D::mcols + c0 + j] = acc[m][j];
        }
    }
    __syncthreads();

    // ---- vertical blur to the moments, S, and the dS/dm maps; a thread owns a run of kRunV rows of one column
    {
        constexpr int kRunV = GRAD ? 5 : 4;  // GRAD: 6 runs x 42 columns, one item per thread
        constexpr int runs = (D::mrows + kRunV - 1) / kRunV;
        for (int it = tid; it < D::mcols * runs; it += kThreads) {
            const int c = it % D::mcols, r0 = (it / D::mcols) * kRunV;
            float mom[5][kRunV];
#pragma unroll
            for (int m = 0; m < 5; m++) {
                float v[kRunV + 2 * kR];
#pragma unroll
                for (int k = 0; k < kRunV + 2 * kR; k++)  // rows past the last run are clamped: their outputs are dropped
                    v[k] = hm[(m * D::hrows + min(r0 + k, D::hrows - 1)) * D::mcols + c];
#pragma unroll
                for (int j = 0; j < kRunV; j++) {
                    float a = 0.f;
#pragma unroll
                    for (int t = 0; t < kTaps; t++) a = fmaf(win.w[t], v[j + t], a);
                    mom[m][j] = a;
                }
            }
            const int gx = tx0 - D::halo + c;
#pragma unroll
            for (int j = 0; j < kRunV; j++) {
                const int r = r0 + j;
                if (r >= D::mrows) break;
                const int gy = ty0 - D::halo + r;
                const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
                const float mx = mom[0][j], my = mom[1][j];
                const float mx2 = mx * mx, my2 = my * my, mxy_ = mx * my;
                const float A1 = 2.f * mxy_ + kC1;
                const float A2 = 2.f * (mom[4][j] - mxy_) + kC2;
                const float B1 = mx2 + my2 + kC1;
                const float B2 = (mom[2][j] - mx2) + (mom[3][j] - my2) + kC2;
                // one division: with iB = 1 / (B1 B2), S/A1 = A2 iB, S/A2 = A1 iB, 1/B2 = B1 iB, 1/B2 - 1/B1 = (B1 - B2) iB
                // (7 divisions per position took 12% more kernel time at 3x1080x1920 on an H100)
                const float iB = 1.f / (B1 * B2);
                const float S = A1 * A2 * iB;
                if (r >= D::halo && r < D::halo + kTY && c >= D::halo && c < D::halo + kTX)
                    s_map[(r - D::halo) * kTX + c - D::halo] = S;
                if (GRAD) {
                    float d0 = 0.f, d1 = 0.f, d2 = 0.f;
                    if (in) {
                        d0 = 2.f * iB * (my * (A2 - A1) + mx * S * (B1 - B2));
                        d1 = -S * B1 * iB;
                        d2 = 2.f * A1 * iB;
                    }
                    dm[(0 * D::mrows + r) * D::mcols + c] = d0;
                    dm[(1 * D::mrows + r) * D::mcols + c] = d1;
                    dm[(2 * D::mrows + r) * D::mcols + c] = d2;
                }
            }
        }
    }

    // ---- GRAD: blur the three maps back to the tile; a warp owns two output rows, lanes consecutive columns
    constexpr int kRowsPerWarp = kTY / (kThreads / 32);
    static_assert(kRowsPerWarp * (kThreads / 32) == kTY && kTX == 32, "a warp row is one tile row");
    const int lane = tid & 31, ry0 = (tid >> 5) * kRowsPerWarp;
    float bd[3][kRowsPerWarp];
    __syncthreads();
    if (GRAD) {
        constexpr int kRunH = 4;
        constexpr int runs = kTX / kRunH;
        for (int it = tid; it < D::mrows * runs; it += kThreads) {
            const int r = it / runs, c0 = (it - r * runs) * kRunH;
#pragma unroll
            for (int m = 0; m < 3; m++) {
                const float* p = dm + (m * D::mrows + r) * D::mcols + c0;
                float v[kRunH + 2 * kR];
#pragma unroll
                for (int k = 0; k < kRunH + 2 * kR; k++) v[k] = p[k];
#pragma unroll
                for (int j = 0; j < kRunH; j++) {
                    float a = 0.f;
#pragma unroll
                    for (int t = 0; t < kTaps; t++) a = fmaf(win.w[t], v[j + t], a);
                    hd[(m * D::mrows + r) * kTX + c0 + j] = a;
                }
            }
        }
        __syncthreads();
#pragma unroll
        for (int m = 0; m < 3; m++) {
            float v[kRowsPerWarp + 2 * kR];
#pragma unroll
            for (int k = 0; k < kRowsPerWarp + 2 * kR; k++) v[k] = hd[(m * D::mrows + ry0 + k) * kTX + lane];
#pragma unroll
            for (int j = 0; j < kRowsPerWarp; j++) {
                float a = 0.f;
#pragma unroll
                for (int t = 0; t < kTaps; t++) a = fmaf(win.w[t], v[j + t], a);
                bd[m][j] = a;
            }
        }
    }

    // ---- L1 term, SSIM sum and the gradient of this thread's kRowsPerWarp pixels
    float l1_sum = 0.f, s_sum = 0.f;
    const int gx = tx0 + lane;
#pragma unroll
    for (int j = 0; j < kRowsPerWarp; j++) {
        const int gy = ty0 + ry0 + j;
        if (gy >= H || gx >= W) continue;
        const int si = (ry0 + j + 2 * kR) * kSX + lane + 2 * kR;
        const float x = sx[si], y = sy[si], d = x - y;
        l1_sum += fabsf(d);
        s_sum += s_map[(ry0 + j) * kTX + lane];
        if (GRAD) {
            const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
            const float gs = bd[0][j] + 2.f * x * bd[1][j] + y * bd[2][j];
            dL_dimage[plane + (size_t)gy * W + gx] = fmaf(w_l1, sgn, w_ssim * gs);
        }
    }

    // ---- per-CTA partial sums, fixed reduction order
    __shared__ float2 red[kThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        l1_sum += __shfl_xor_sync(0xffffffffu, l1_sum, o);
        s_sum += __shfl_xor_sync(0xffffffffu, s_sum, o);
    }
    if (lane == 0) red[tid >> 5] = make_float2(l1_sum, s_sum);
    __syncthreads();
    if (tid == 0) {
        float2 t = red[0];
        for (int w = 1; w < kThreads / 32; w++) {
            t.x += red[w].x;
            t.y += red[w].y;
        }
        partial[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = t;
    }
}

// One CTA sums the per-CTA partials in double, each thread a fixed strided subset, then a fixed tree.
constexpr int kReduceThreads = 512;

__global__ void __launch_bounds__(kReduceThreads) image_loss_reduce_kernel(const float2* __restrict__ partial, size_t n,
                                                                            float* __restrict__ sums) {
    __shared__ double r0[kReduceThreads], r1[kReduceThreads];
    double a = 0.0, b = 0.0;
    for (size_t i = threadIdx.x; i < n; i += kReduceThreads) {
        const float2 p = partial[i];
        a += p.x;
        b += p.y;
    }
    r0[threadIdx.x] = a;
    r1[threadIdx.x] = b;
    __syncthreads();
    for (int s = kReduceThreads / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            r0[threadIdx.x] += r0[threadIdx.x + s];
            r1[threadIdx.x] += r1[threadIdx.x + s];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        sums[0] = (float)r0[0];
        sums[1] = (float)r1[0];
    }
}

Window gaussian_window() {  // utils/loss_utils.py gaussian(11, 1.5): exp(-(i - 5)^2 / 4.5), normalised to sum 1
    double g[kTaps], s = 0.0;
    for (int i = 0; i < kTaps; i++) s += (g[i] = std::exp(-(double)((i - kR) * (i - kR)) / 4.5));
    Window w;
    for (int i = 0; i < kTaps; i++) w.w[i] = (float)(g[i] / s);
    return w;
}

template <bool GRAD>
cudaError_t launch(dim3 grid, int H, int W, const float* image, const float* gt, float w_l1, float w_ssim,
                   float2* partial, float* dL_dimage, cudaStream_t s) {
    const size_t smem = Dims<GRAD>::smem_floats * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(image_loss_kernel<GRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    image_loss_kernel<GRAD><<<grid, kThreads, smem, s>>>(H, W, gaussian_window(), image, gt, w_l1, w_ssim, partial,
                                                          dL_dimage);
    return cudaGetLastError();
}

}  // namespace

bool image_loss_grid_ok(int planes, int H, int W) {
    return planes <= 65535 && (H + kTY - 1) / kTY <= 65535 && W <= 0x7fffffff - kTX;
}

cudaError_t launch_image_loss(int planes, int H, int W, const float* image, const float* gt, float w_l1, float w_ssim,
                              float* sums, float* dL_dimage, cudaStream_t s) {
    if (planes == 0) return cudaSuccess;
    if (!image_loss_grid_ok(planes, H, W)) return cudaErrorInvalidValue;
    const dim3 grid((W + kTX - 1) / kTX, (H + kTY - 1) / kTY, planes);
    const size_t n = (size_t)grid.x * grid.y * grid.z;
    float2* partial = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&partial, n * sizeof(float2), s);
    if (e != cudaSuccess) return e;
    e = dL_dimage ? launch<true>(grid, H, W, image, gt, w_l1, w_ssim, partial, dL_dimage, s)
                  : launch<false>(grid, H, W, image, gt, w_l1, w_ssim, partial, nullptr, s);
    if (e == cudaSuccess) {
        image_loss_reduce_kernel<<<1, kReduceThreads, 0, s>>>(partial, n, sums);
        e = cudaGetLastError();
        g_launches += 2;
    }
    cudaFreeAsync(partial, s);
    return e;
}

}  // namespace f3dgs
