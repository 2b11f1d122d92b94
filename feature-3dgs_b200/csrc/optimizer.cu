// Activation prologue and fused optimizer step on the replicated parameter buffers (SURVEY.md section 8 f3 / f2).
//
// Reference (scene/gaussian_model.py):
//   :98-121   get_scaling = exp(_scaling), get_rotation = normalize(_rotation), get_opacity = sigmoid(_opacity),
//             get_features = cat(_features_dc, _features_rest) -- four elementwise PyTorch kernels and a 192-byte-per-
//             Gaussian concat per view, plus their autograd backward kernels;
//   :163-190  torch.optim.Adam(lr=0, eps=1e-15) over seven parameter groups with their own learning rates.
// Here:
//   activate_*        one pass: raw parameters -> the activated tensors the rasterizer consumes (once per optimizer step, not
//                     per view: the parameters do not change between the views of a step);
//   adam_step_kernel  one pass per group: takes the gradient w.r.t. the ACTIVATED tensor (what the rasterizer's backward
//                     accumulates in the flat buffer, after the all-reduce), applies the activation's Jacobian
//                     (sigmoid / exp / normalize / the dc-rest split of the SH tensor) and the Adam update in place.
//                     Formulas follow torch.optim.Adam's single-tensor path: m <- lerp(m, g, 1 - b1),
//                     v <- b2 v + (1 - b2) g^2, p <- p - (lr / (1 - b1^t)) m / (sqrt(v) / sqrt(1 - b2^t) + eps).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/f3dgs_b200.h"
#include "kernels.h"

namespace f3dgs {
namespace {

__global__ void __launch_bounds__(256) activate_kernel(int P, int M, const float* __restrict__ raw_opacity,
                                                       const float* __restrict__ raw_scaling,
                                                       const float* __restrict__ raw_rotation,
                                                       const float* __restrict__ f_dc, const float* __restrict__ f_rest,
                                                       float* __restrict__ opacity, float* __restrict__ scales,
                                                       float* __restrict__ rotations, float* __restrict__ shs) {
    // flat work list: [0, P) opacity | [P, 4P) scales | [4P, 5P) rotations (one float4 each) | [5P, 5P + 3MP) SH concat
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n_op = (size_t)P, n_sc = 3 * (size_t)P, n_rot = (size_t)P, n_sh = 3 * (size_t)M * P;
    if (i < n_op) {
        if (raw_opacity) opacity[i] = 1.0f / (1.0f + expf(-raw_opacity[i]));  // torch.sigmoid
    } else if (i < n_op + n_sc) {
        const size_t j = i - n_op;
        if (raw_scaling) scales[j] = expf(raw_scaling[j]);
    } else if (i < n_op + n_sc + n_rot) {
        const size_t j = i - n_op - n_sc;
        if (raw_rotation) {
            const float4 q = reinterpret_cast<const float4*>(raw_rotation)[j];
            const float nrm = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);  // F.normalize eps
            reinterpret_cast<float4*>(rotations)[j] = make_float4(q.x / nrm, q.y / nrm, q.z / nrm, q.w / nrm);
        }
    } else if (i < n_op + n_sc + n_rot + n_sh) {
        const size_t j = i - n_op - n_sc - n_rot;
        if (f_dc) {
            const size_t p = j / (3 * (size_t)M), e = j % (3 * (size_t)M);
            shs[j] = e < 3 ? f_dc[3 * p + e] : f_rest[p * 3 * (size_t)(M - 1) + (e - 3)];
        }
    }
}

struct AdamArgs {
    float* param;        // raw parameter, updated in place
    const float* grad;   // gradient w.r.t. the activated tensor (layout of the activated tensor)
    float* m;
    float* v;
    size_t n;            // elements of the raw parameter
    int kind, M;
    float lr_over_bc1, inv_sqrt_bc2, b1, b2, eps;
};

__device__ __forceinline__ void adam_update(float& p, float& m, float& v, float g, const AdamArgs& a) {
    m = m + (1.0f - a.b1) * (g - m);
    v = v * a.b2 + (1.0f - a.b2) * g * g;
    const float denom = sqrtf(v) * a.inv_sqrt_bc2 + a.eps;
    p = p - a.lr_over_bc1 * (m / denom);
}

__global__ void __launch_bounds__(256) adam_step_kernel(AdamArgs a) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a.kind == F3DGS_PARAM_NORMALIZE4) {
        if (i >= a.n / 4) return;
        float4 r = reinterpret_cast<float4*>(a.param)[i];
        const float4 g = reinterpret_cast<const float4*>(a.grad)[i];
        const float nrm = fmaxf(sqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w), 1e-12f);
        const float4 q = make_float4(r.x / nrm, r.y / nrm, r.z / nrm, r.w / nrm);
        const float qg = q.x * g.x + q.y * g.y + q.z * g.z + q.w * g.w;
        const float4 dr = make_float4((g.x - q.x * qg) / nrm, (g.y - q.y * qg) / nrm, (g.z - q.z * qg) / nrm,
                                      (g.w - q.w * qg) / nrm);
        float4 m = reinterpret_cast<float4*>(a.m)[i], v = reinterpret_cast<float4*>(a.v)[i];
        adam_update(r.x, m.x, v.x, dr.x, a);
        adam_update(r.y, m.y, v.y, dr.y, a);
        adam_update(r.z, m.z, v.z, dr.z, a);
        adam_update(r.w, m.w, v.w, dr.w, a);
        reinterpret_cast<float4*>(a.param)[i] = r;
        reinterpret_cast<float4*>(a.m)[i] = m;
        reinterpret_cast<float4*>(a.v)[i] = v;
        return;
    }
    if (i >= a.n) return;
    float p = a.param[i], g;
    switch (a.kind) {
        case F3DGS_PARAM_SIGMOID: {
            const float o = 1.0f / (1.0f + expf(-p));
            g = a.grad[i] * o * (1.0f - o);
            break;
        }
        case F3DGS_PARAM_EXP: g = a.grad[i] * expf(p); break;
        case F3DGS_PARAM_SH_DC: g = a.grad[(i / 3) * 3 * (size_t)a.M + (i % 3)]; break;
        case F3DGS_PARAM_SH_REST: {
            const size_t per = 3 * (size_t)(a.M - 1);
            g = a.grad[(i / per) * 3 * (size_t)a.M + 3 + (i % per)];
            break;
        }
        default: g = a.grad[i]; break;
    }
    float m = a.m[i], v = a.v[i];
    adam_update(p, m, v, g, a);
    a.param[i] = p;
    a.m[i] = m;
    a.v[i] = v;
}

}  // namespace

cudaError_t launch_activate(int P, int M, const float* raw_opacity, const float* raw_scaling, const float* raw_rotation,
                            const float* features_dc, const float* features_rest, float* opacity, float* scales,
                            float* rotations, float* shs, cudaStream_t s) {
    const size_t n = 5 * (size_t)P + 3 * (size_t)M * P;
    activate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(P, M, raw_opacity, raw_scaling, raw_rotation, features_dc,
                                                                features_rest, opacity, scales, rotations, shs);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_adam_step(int kind, size_t n, int M, float* param, const float* grad_activated, float* exp_avg,
                             float* exp_avg_sq, float lr, float beta1, float beta2, float eps, int step, cudaStream_t s) {
    AdamArgs a;
    a.param = param; a.grad = grad_activated; a.m = exp_avg; a.v = exp_avg_sq; a.n = n; a.kind = kind; a.M = M;
    const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    a.lr_over_bc1 = (float)((double)lr / bc1);
    a.inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
    a.b1 = beta1; a.b2 = beta2; a.eps = eps;
    const size_t threads = kind == F3DGS_PARAM_NORMALIZE4 ? n / 4 : n;
    adam_step_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(a);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace f3dgs
