// Per-Gaussian front end and back end of the splat pipeline (streaming, one thread per Gaussian).
//
//   preprocess_fwd_kernel  : reference FORWARD::preprocessCUDA, forward.cu:156-256
//                            (+ computeCov3D :119-153, computeCov2D :75-114, computeColorFromSH :20-72,
//                               in_frustum auxiliary.h:145-170, getRect :46-56, ndc2Pix :41-44)
//   preprocess_bwd_kernel  : reference computeCov2DCUDA backward.cu:144-274 fused with
//                            BACKWARD::preprocessCUDA :346-404 (computeColorFromSH bwd :20-139,
//                            computeCov3D bwd :278-341)
//   mark_visible_kernel    : reference checkFrustum, rasterizer_impl.cu:54-66
//
// The forward kernel reproduces the reference's fp32 operation sequence exactly (see common.cuh),
// because radii, tile rectangles and depth bits feed the bit-exact tile/key contract.
#include <cstdio>

#include "kernels.h"

namespace f3dgs {

__device__ __constant__ float kSH_C0 = 0.28209479177387814f;
__device__ __constant__ float kSH_C1 = 0.4886025119029199f;
__device__ __constant__ float kSH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                           -1.0925484305920792f, 0.5462742152960396f};
__device__ __constant__ float kSH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                           0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                                           -0.5900435899266435f};

struct F3 {
    float x, y, z;
};
__device__ __forceinline__ F3 operator+(F3 a, F3 b) { return F3{a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ F3 operator-(F3 a, F3 b) { return F3{a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ F3 operator*(float s, F3 a) { return F3{s * a.x, s * a.y, s * a.z}; }
__device__ __forceinline__ F3 operator/(F3 a, float s) { return F3{a.x / s, a.y / s, a.z / s}; }

// Column-major 3x3 (c[col][row]) with the same product expansion as the matrix library the
// reference uses (GLM 0.9.9, type_mat3x3.inl:486-519): element (col j,row i) of A*B is
// A[0][i]*B[j][0] + A[1][i]*B[j][1] + A[2][i]*B[j][2], summed left to right.  Keeping the same
// expression tree (zero terms included) is what makes nvcc place the same FMAs as in the reference.
struct M3 {
    float c[3][3];
};
__device__ __forceinline__ M3 operator*(const M3& A, const M3& B) {
    M3 R;
#pragma unroll
    for (int j = 0; j < 3; j++)
#pragma unroll
        for (int i = 0; i < 3; i++) R.c[j][i] = A.c[0][i] * B.c[j][0] + A.c[1][i] * B.c[j][1] + A.c[2][i] * B.c[j][2];
    return R;
}
__device__ __forceinline__ M3 transpose(const M3& A) {
    M3 R;
#pragma unroll
    for (int j = 0; j < 3; j++)
#pragma unroll
        for (int i = 0; i < 3; i++) R.c[j][i] = A.c[i][j];
    return R;
}
__device__ __forceinline__ M3 cols(float a0, float a1, float a2, float b0, float b1, float b2, float c0, float c1,
                                   float c2) {
    M3 R;
    R.c[0][0] = a0; R.c[0][1] = a1; R.c[0][2] = a2;
    R.c[1][0] = b0; R.c[1][1] = b1; R.c[1][2] = b2;
    R.c[2][0] = c0; R.c[2][1] = c1; R.c[2][2] = c2;
    return R;
}

// reference auxiliary.h:58-77: rows of the column-major 4x4 applied to a point
__device__ __forceinline__ float xf(const float* __restrict__ m, int r, F3 p) {
    return m[r] * p.x + m[4 + r] * p.y + m[8 + r] * p.z + m[12 + r];
}

// SH -> RGB, reference forward.cu:20-72.  `sh` points at this Gaussian's [M,3] coefficients.
__device__ __forceinline__ F3 sh_to_rgb(int deg, const float* __restrict__ shp, F3 pos, const float* __restrict__ cam,
                                        uint8_t& clamp_bits) {
    const F3* sh = reinterpret_cast<const F3*>(shp);
    F3 dir = pos - F3{cam[0], cam[1], cam[2]};
    const F3 sq = F3{dir.x * dir.x, dir.y * dir.y, dir.z * dir.z};
    dir = dir / sqrtf(sq.x + sq.y + sq.z);
    F3 result = kSH_C0 * sh[0];
    if (deg > 0) {
        const float x = dir.x, y = dir.y, z = dir.z;
        result = result - kSH_C1 * y * sh[1] + kSH_C1 * z * sh[2] - kSH_C1 * x * sh[3];
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z;
            const float xy = x * y, yz = y * z, xz = x * z;
            result = result + kSH_C2[0] * xy * sh[4] + kSH_C2[1] * yz * sh[5] +
                     kSH_C2[2] * (2.0f * zz - xx - yy) * sh[6] + kSH_C2[3] * xz * sh[7] +
                     kSH_C2[4] * (xx - yy) * sh[8];
            if (deg > 2) {
                result = result + kSH_C3[0] * y * (3.0f * xx - yy) * sh[9] + kSH_C3[1] * xy * z * sh[10] +
                         kSH_C3[2] * y * (4.0f * zz - xx - yy) * sh[11] +
                         kSH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh[12] +
                         kSH_C3[4] * x * (4.0f * zz - xx - yy) * sh[13] + kSH_C3[5] * z * (xx - yy) * sh[14] +
                         kSH_C3[6] * x * (xx - 3.0f * yy) * sh[15];
            }
        }
    }
    result.x += 0.5f;
    result.y += 0.5f;
    result.z += 0.5f;
    clamp_bits = (result.x < 0 ? 1 : 0) | (result.y < 0 ? 2 : 0) | (result.z < 0 ? 4 : 0);
    return F3{fmaxf(result.x, 0.0f), fmaxf(result.y, 0.0f), fmaxf(result.z, 0.0f)};
}

// scale/rotation -> world covariance (upper triangle), reference forward.cu:119-153
__device__ __forceinline__ void cov3d_from_scale_rot(const float* __restrict__ s3, float mod,
                                                     const float* __restrict__ q4, float* cov) {
    M3 S = cols(1.0f, 0.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.0f, 1.0f);
    S.c[0][0] = mod * s3[0];
    S.c[1][1] = mod * s3[1];
    S.c[2][2] = mod * s3[2];
    const float r = q4[0], x = q4[1], y = q4[2], z = q4[3];  // not renormalised (forward.cu:128)
    const M3 R = cols(1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y),
                      2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x),
                      2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y));
    const M3 M = S * R;
    const M3 Sigma = transpose(M) * M;
    cov[0] = Sigma.c[0][0];
    cov[1] = Sigma.c[0][1];
    cov[2] = Sigma.c[0][2];
    cov[3] = Sigma.c[1][1];
    cov[4] = Sigma.c[1][2];
    cov[5] = Sigma.c[2][2];
}

// EWA projection of the 3-D covariance, reference forward.cu:75-114.  Returns (a, b, c) with the
// 0.3 dilation applied, and the undilated diagonal (a0, c0) for antialiasing.  Also hands back the intermediates the
// backward needs.
struct Cov2D {
    float a, b, c;
    float a0, c0;
    float T00, T01, T02, T10, T11, T12;  // T[0][*], T[1][*] of T = W * J (column-major indexing)
    float tx, ty, tz;                    // clamped view-space mean
    float txtz, tytz;                    // unclamped ratios
};
__device__ __forceinline__ Cov2D project_cov(F3 mean, const float* __restrict__ vm, float focal_x, float focal_y,
                                             float tan_fovx, float tan_fovy, const float* __restrict__ cv) {
    Cov2D o;
    F3 t = F3{xf(vm, 0, mean), xf(vm, 1, mean), xf(vm, 2, mean)};
    const float limx = 1.3f * tan_fovx;
    const float limy = 1.3f * tan_fovy;
    const float txtz = t.x / t.z;
    const float tytz = t.y / t.z;
    t.x = fminf(limx, fmaxf(-limx, txtz)) * t.z;
    t.y = fminf(limy, fmaxf(-limy, tytz)) * t.z;
    const M3 J = cols(focal_x / t.z, 0.0f, -(focal_x * t.x) / (t.z * t.z), 0.0f, focal_y / t.z,
                      -(focal_y * t.y) / (t.z * t.z), 0.0f, 0.0f, 0.0f);
    const M3 Wm = cols(vm[0], vm[4], vm[8], vm[1], vm[5], vm[9], vm[2], vm[6], vm[10]);
    const M3 T = Wm * J;
    const M3 Vrk = cols(cv[0], cv[1], cv[2], cv[1], cv[3], cv[4], cv[2], cv[4], cv[5]);
    M3 cov = transpose(T) * transpose(Vrk) * T;
    o.a0 = cov.c[0][0]; o.c0 = cov.c[1][1];
    cov.c[0][0] += 0.3f;
    cov.c[1][1] += 0.3f;
    o.a = cov.c[0][0]; o.b = cov.c[0][1]; o.c = cov.c[1][1];
    o.T00 = T.c[0][0]; o.T01 = T.c[0][1]; o.T02 = T.c[0][2];
    o.T10 = T.c[1][0]; o.T11 = T.c[1][1]; o.T12 = T.c[1][2];
    o.tx = t.x; o.ty = t.y; o.tz = t.z; o.txtz = txtz; o.tytz = tytz;
    return o;
}

// Conservative half extents of {d : opacity * exp(-0.5 d^T Q d) >= 1/255}, Q = conic.
// Used only to skip (pixel block, Gaussian) pairs the blend would reject anyway
// (reference forward.cu:352 `alpha < 1/255 -> continue`), so it never changes a result.
__device__ __forceinline__ void alpha_extent(float A, float B, float C, float op, float& ex, float& ey) {
    if (!(op >= 1.0f / 255.0f)) {  // G <= 1  =>  alpha <= op < 1/255 for every pixel
        ex = ey = -3.0e38f;  // x + ex >= lo is false for every block
        return;
    }
    const float ac = A * C;
    const float det = ac - B * B;
    if (!(A > 0.f) || !(C > 0.f) || !(det > 1e-4f * ac) || !(det < 3.0e38f)) {
        ex = ey = 3.0e38f;  // ill-conditioned or indefinite conic: never cull
        return;
    }
    const float tau = 2.02f * __logf(255.0f * op) + 0.02f;  // 2 ln(255 op), inflated by > 1 %
    ex = sqrtf(tau * C / det) + 0.01f;
    ey = sqrtf(tau * A / det) + 0.01f;
}

// Antialiasing (AA = true): the 0.3 px^2 dilation widens a Gaussian without conserving its integral, so the opacity is
// scaled by rho = sqrt(max(kAaMinRatio, det0 / det)), det0 = a0 c0 - b^2 of the undilated and det = a c - b^2 of the
// dilated 2-D covariance; the dilated splat then carries the undilated one's integral.  The ratio is formed from opaque
// copies of its inputs, so that sharing a product with `det` cannot change how the compiler contracts the default
// path's arithmetic: conic, radius and everything else keep the bits of AA = false.
constexpr float kAaMinRatio = 2.5e-5f;
__device__ __forceinline__ float aa_det0(float a0, float b, float c0) {
    asm("" : "+f"(a0), "+f"(b), "+f"(c0));
    return a0 * c0 - b * b;
}

// shared-memory staging of SH rows (both preprocess kernels)
constexpr int kBwdBlock = 128;
__host__ __device__ constexpr int bwd_row_stride(int row_floats) { return row_floats | 1; }  // odd stride: no bank conflicts

template <bool AA>
__global__ void __launch_bounds__(256)
preprocess_fwd_kernel(ViewParams vp, const float* __restrict__ means3D, const float* __restrict__ scales,
                      const float* __restrict__ rotations, const float* __restrict__ opacities,
                      const float* __restrict__ shs, const float* __restrict__ cov3D_precomp,
                      const float* __restrict__ colors_precomp, bool prefiltered, int* __restrict__ radii,
                      SplatRec* __restrict__ rec, float* __restrict__ cov3D, uint8_t* __restrict__ clamped,
                      uint32_t* __restrict__ tiles_touched) {
    // SH rows (12 M bytes per Gaussian) come in through shared memory with coalesced 128-bit loads; each thread then reads
    // its own padded row (see preprocess_bwd_kernel).  The arithmetic on the values is unchanged.
    extern __shared__ float fwd_sh_rows[];
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int row_floats = vp.M * 3, stride = bwd_row_stride(row_floats);
    if (shs != nullptr) {
        const int block_base = blockIdx.x * blockDim.x;
        const int rows_here = min((int)blockDim.x, vp.P - block_base);
        const float* src = shs + (size_t)block_base * row_floats;
        if ((row_floats & 3) == 0 && (reinterpret_cast<uintptr_t>(shs) & 15) == 0) {
            const int q_per_row = row_floats >> 2;
            for (int i = threadIdx.x; i < rows_here * q_per_row; i += blockDim.x) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(src) + i);
                float* d = fwd_sh_rows + (i / q_per_row) * stride + (i % q_per_row) * 4;
                d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
            }
        } else {
            for (int i = threadIdx.x; i < rows_here * row_floats; i += blockDim.x)
                fwd_sh_rows[(i / row_floats) * stride + (i % row_floats)] = __ldg(src + i);
        }
        __syncthreads();
    }
    if (idx >= vp.P) return;
    int my_radii = 0;
    uint32_t my_tiles = 0;
    do {
        const F3 p_orig = F3{means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]};
        const float* vm = vp.viewmatrix;
        const float* pm = vp.projmatrix;
        const float depth = xf(vm, 2, p_orig);
        if (depth <= 0.2f) {  // reference auxiliary.h:160 (only the near plane culls)
            if (prefiltered) {
                printf("Point is filtered although prefiltered is set. This shouldn't happen!");
                __trap();
            }
            break;
        }
        const float hx = xf(pm, 0, p_orig), hy = xf(pm, 1, p_orig), hw = xf(pm, 3, p_orig);
        const float p_w = 1.0f / (hw + 0.0000001f);
        const float projx = hx * p_w, projy = hy * p_w;

        float cv[6];
        if (cov3D_precomp != nullptr) {
#pragma unroll
            for (int i = 0; i < 6; i++) cv[i] = cov3D_precomp[6 * idx + i];
        } else {
            cov3d_from_scale_rot(scales + 3 * idx, vp.scale_modifier, rotations + 4 * idx, cv);
#pragma unroll
            for (int i = 0; i < 6; i++) cov3D[6 * idx + i] = cv[i];
        }
        const Cov2D c2 = project_cov(p_orig, vm, vp.focal_x, vp.focal_y, vp.tan_fovx, vp.tan_fovy, cv);
        const float det = (c2.a * c2.c - c2.b * c2.b);
        if (det == 0.0f) break;
        const float det_inv = 1.f / det;
        const float conA = c2.c * det_inv, conB = -c2.b * det_inv, conC = c2.a * det_inv;
        const float mid = 0.5f * (c2.a + c2.c);
        const float lambda1 = mid + sqrtf(fmaxf(0.1f, mid * mid - det));
        const float lambda2 = mid - sqrtf(fmaxf(0.1f, mid * mid - det));
        const float rad_f = ceilf(3.f * sqrtf(fmaxf(lambda1, lambda2)));
        const int rad = (int)rad_f;
        const float ix = ndc2pix(projx, vp.W), iy = ndc2pix(projy, vp.H);
        uint32_t x0, y0, x1, y1;
        tile_rect(ix, iy, rad, vp.grid_x, vp.grid_y, x0, y0, x1, y1);
        const uint32_t area = (x1 - x0) * (y1 - y0);
        if (area == 0) break;

        SplatRec r;
        uint8_t cb = 0;
        if (colors_precomp == nullptr) {
            F3 col = sh_to_rgb(vp.D, fwd_sh_rows + threadIdx.x * stride, p_orig, vp.cam_pos, cb);
            r.r = col.x; r.g = col.y; r.b = col.z;
        } else {
            r.r = colors_precomp[3 * idx]; r.g = colors_precomp[3 * idx + 1]; r.b = colors_precomp[3 * idx + 2];
        }
        clamped[idx] = cb;
        r.x = ix; r.y = iy;
        r.ca = conA; r.cb = conB; r.cc = conC;
        r.op = opacities[idx];
        if constexpr (AA) r.op *= sqrtf(fmaxf(kAaMinRatio, aa_det0(c2.a0, c2.b, c2.c0) / det));
        r.depth = depth;
#ifdef F3DGS_SASS_AUDIT  // build used only to compare the FP instruction mix with the reference kernel
        r.ex = r.ey = 0.f;
#else
        alpha_extent(conA, conB, conC, r.op, r.ex, r.ey);
#endif
        float4* dst = reinterpret_cast<float4*>(rec + idx);
        dst[0] = make_float4(r.x, r.y, r.ex, r.ey);
        dst[1] = make_float4(r.ca, r.cb, r.cc, r.op);
        dst[2] = make_float4(r.r, r.g, r.b, r.depth);
        my_radii = rad;
        my_tiles = area;
    } while (false);
    radii[idx] = my_radii;
    tiles_touched[idx] = my_tiles;
}

__global__ void __launch_bounds__(256)
mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ vm,
                    uint8_t* __restrict__ present) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float z = xf(vm, 2, F3{means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]});
    present[idx] = z > 0.2f ? 1 : 0;
}

// -------------------------------------------------------------------------------- backward
__device__ __forceinline__ F3 dnormvdv3(F3 v, F3 dv) {  // reference auxiliary.h:107-117
    const float sum2 = v.x * v.x + v.y * v.y + v.z * v.z;
    const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
    F3 o;
    o.x = ((+sum2 - v.x * v.x) * dv.x - v.y * v.x * dv.y - v.z * v.x * dv.z) * invsum32;
    o.y = (-v.x * v.y * dv.x + (sum2 - v.y * v.y) * dv.y - v.z * v.y * dv.z) * invsum32;
    o.z = (-v.x * v.z * dv.x - v.y * v.z * dv.y + (sum2 - v.z * v.z) * dv.z) * invsum32;
    return o;
}

// SH backward of one Gaussian (reference backward.cu:20-139): writes the coefficient gradients dsh (dRGB: the colour
// gradient, 0 on clamped channels) for the unit view direction (x, y, z) and returns dL/d(x, y, z).
__device__ __forceinline__ F3 sh_dir_grad(int deg, const float* sh, float* dsh, const float (&dRGB)[3], float x, float y,
                                          float z) {
    float ddx = 0.f, ddy = 0.f, ddz = 0.f;  // dL/ddir
#define SHC(k, c) sh[3 * (k) + (c)]
#define WR(k, coef)                                                  \
    do {                                                             \
    const float cf_ = (coef);                                    \
    dsh[3 * (k)] = cf_ * dRGB[0];                                \
    dsh[3 * (k) + 1] = cf_ * dRGB[1];                            \
    dsh[3 * (k) + 2] = cf_ * dRGB[2];                            \
    } while (0)
    WR(0, kSH_C0);
    if (deg > 0) {
        WR(1, -kSH_C1 * y);
        WR(2, kSH_C1 * z);
        WR(3, -kSH_C1 * x);
        float dx_[3], dy_[3], dz_[3];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
            dx_[ch] = -kSH_C1 * SHC(3, ch);
            dy_[ch] = -kSH_C1 * SHC(1, ch);
            dz_[ch] = kSH_C1 * SHC(2, ch);
        }
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z;
            const float xy = x * y, yz = y * z, xz = x * z;
            WR(4, kSH_C2[0] * xy);
            WR(5, kSH_C2[1] * yz);
            WR(6, kSH_C2[2] * (2.f * zz - xx - yy));
            WR(7, kSH_C2[3] * xz);
            WR(8, kSH_C2[4] * (xx - yy));
#pragma unroll
            for (int ch = 0; ch < 3; ch++) {
                dx_[ch] += kSH_C2[0] * y * SHC(4, ch) + kSH_C2[2] * 2.f * -x * SHC(6, ch) +
                           kSH_C2[3] * z * SHC(7, ch) + kSH_C2[4] * 2.f * x * SHC(8, ch);
                dy_[ch] += kSH_C2[0] * x * SHC(4, ch) + kSH_C2[1] * z * SHC(5, ch) +
                           kSH_C2[2] * 2.f * -y * SHC(6, ch) + kSH_C2[4] * 2.f * -y * SHC(8, ch);
                dz_[ch] += kSH_C2[1] * y * SHC(5, ch) + kSH_C2[2] * 2.f * 2.f * z * SHC(6, ch) +
                           kSH_C2[3] * x * SHC(7, ch);
            }
            if (deg > 2) {
                WR(9, kSH_C3[0] * y * (3.f * xx - yy));
                WR(10, kSH_C3[1] * xy * z);
                WR(11, kSH_C3[2] * y * (4.f * zz - xx - yy));
                WR(12, kSH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy));
                WR(13, kSH_C3[4] * x * (4.f * zz - xx - yy));
                WR(14, kSH_C3[5] * z * (xx - yy));
                WR(15, kSH_C3[6] * x * (xx - 3.f * yy));
#pragma unroll
                for (int ch = 0; ch < 3; ch++) {
                    dx_[ch] += (kSH_C3[0] * SHC(9, ch) * 3.f * 2.f * xy + kSH_C3[1] * SHC(10, ch) * yz +
                                kSH_C3[2] * SHC(11, ch) * -2.f * xy + kSH_C3[3] * SHC(12, ch) * -3.f * 2.f * xz +
                                kSH_C3[4] * SHC(13, ch) * (-3.f * xx + 4.f * zz - yy) +
                                kSH_C3[5] * SHC(14, ch) * 2.f * xz + kSH_C3[6] * SHC(15, ch) * 3.f * (xx - yy));
                    dy_[ch] += (kSH_C3[0] * SHC(9, ch) * 3.f * (xx - yy) + kSH_C3[1] * SHC(10, ch) * xz +
                                kSH_C3[2] * SHC(11, ch) * (-3.f * yy + 4.f * zz - xx) +
                                kSH_C3[3] * SHC(12, ch) * -3.f * 2.f * yz + kSH_C3[4] * SHC(13, ch) * -2.f * xy +
                                kSH_C3[5] * SHC(14, ch) * -2.f * yz + kSH_C3[6] * SHC(15, ch) * -3.f * 2.f * xy);
                    dz_[ch] += (kSH_C3[1] * SHC(10, ch) * xy + kSH_C3[2] * SHC(11, ch) * 4.f * 2.f * yz +
                                kSH_C3[3] * SHC(12, ch) * 3.f * (2.f * zz - xx - yy) +
                                kSH_C3[4] * SHC(13, ch) * 4.f * 2.f * xz + kSH_C3[5] * SHC(14, ch) * (xx - yy));
                }
            }
        }
        ddx = dx_[0] * dRGB[0] + dx_[1] * dRGB[1] + dx_[2] * dRGB[2];
        ddy = dy_[0] * dRGB[0] + dy_[1] * dRGB[1] + dy_[2] * dRGB[2];
        ddz = dz_[0] * dRGB[0] + dz_[1] * dRGB[1] + dz_[2] * dRGB[2];
    }
#undef SHC
#undef WR
    return F3{ddx, ddy, ddz};
}

// The antialiased kernels run the SH backward out of line.  Inlined, ptxas fuses its multiplies and adds differently
// in each instantiation, so dL_dsh and dL_dmean3D of the camera and accumulating twins would differ in the last bit;
// one compiled body gives every twin the same bits.  -> dL/dmean through the view direction; *dd = dL/ddir.  (The
// default kernels keep the inline code, whose instructions their twins already share.)
__device__ __noinline__ F3 sh_backward_out_of_line(int deg, const float* sh, float* dsh, float r, float g, float b,
                                                   F3 dir_orig, F3* dd) {
    const float inv_len = 1.0f / sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
    const float dRGB[3] = {r, g, b};
    *dd = sh_dir_grad(deg, sh, dsh, dRGB, dir_orig.x * inv_len, dir_orig.y * inv_len, dir_orig.z * inv_len);
    return dnormvdv3(dir_orig, *dd);
}

// ACCUM = false: the reference's contract -- gradients are ASSIGNED (backward.cu:273, :217-232, :48-97, :323-340) into
// zero-filled buffers.  ACCUM = true (view batches, f3dgs_backward_accum): every per-parameter gradient is ADDED to what
// is already there (each Gaussian is written by exactly one thread: plain read-modify-write, no atomics), and the
// densification statistics of scene/gaussian_model.py:436-438 are folded in.
template <bool ACCUM>
__device__ __forceinline__ void put(float* __restrict__ dst, float v) {
    if (ACCUM) *dst += v;
    else *dst = v;
}

// The 12 M bytes of SH coefficients per Gaussian (192 B at M = 16) are the widest operand of this kernel, read once and --
// as gradients -- written once (read-modify-written in ACCUM mode).  One thread per Gaussian touching its own row gives 32
// rows x 4 bytes per warp instruction, i.e. one useful word per 32-byte sector.  So the block stages both directions in
// shared memory: rows come in and go out with coalesced 128-bit accesses, each thread works on its own (padded,
// conflict-free) row in between.

// Camera gradient (CAM = true).  Each visible Gaussian contributes kCamTerms floats, slot j:
//   j = 3k + r       (k = 0..3, r = 0..2)      dL/dviewmatrix[4k + r]   view-space mean, depth and W of T = W J
//   j = 12 + 3k + i  (k = 0..3, r = 0, 1, 3)  dL/dprojmatrix[4k + r]   screen-space mean
//   j = 24 + k       (k = 0..2)                dL/dcampos[k]            SH view direction
// The other 8 matrix entries (vm[3,7,11,15], pm[2,6,10,14]) are never read by the forward: their gradient is 0.
constexpr int kCamTerms = 27;
__host__ __device__ constexpr int cam_slot(int j) {  // slot -> index in the 35-float camera gradient
    return j < 12 ? 4 * (j / 3) + j % 3
                  : j < 24 ? 16 + 4 * ((j - 12) / 3) + ((j - 12) % 3 == 2 ? 3 : (j - 12) % 3) : 32 + (j - 24);
}

// AA = true: the backward of the antialiased forward.  The composite's opacity gradient g = dL/dop_eff is read from
// dL_dop_eff; dL_dopacity gets rho g (assigned or added, as every other gradient), and rho's dependence on the 2-D
// covariance joins dL/d(a, b, c), from where it reaches cov3D, scale, rotation, the mean and the camera.  op_eff is the
// splat record's op.  dL_dop_eff may be dL_dopacity itself (the assigning backward rescales in place): the two are read
// and written by the same thread, so neither is __restrict__.
// ABS = true (ACCUM only): AbsGS's statistic grad_accum_abs += ||dL_dmean2D_abs.xy||, gated and formed as grad_accum is.
template <bool ACCUM, bool CAM, bool AA, bool ABS = false>
__global__ void __launch_bounds__(kBwdBlock)
preprocess_bwd_kernel(ViewParams vp, const float* __restrict__ means3D, const int* __restrict__ radii,
                      const float* __restrict__ shs, const uint8_t* __restrict__ clamped,
                      const float* __restrict__ scales, const float* __restrict__ rotations,
                      const float* __restrict__ cov3D, const float* __restrict__ dL_dmean2D,
                      const float* __restrict__ dL_dconic, float* __restrict__ dL_dmean3D,
                      const float* __restrict__ dL_dcolor, float* __restrict__ dL_dcov3D,
                      float* __restrict__ dL_dsh, float* __restrict__ dL_dscale, float* __restrict__ dL_drot,
                      const float* __restrict__ dL_dz, float* __restrict__ grad_accum, float* __restrict__ vis_count,
                      double* __restrict__ cam_part, const SplatRec* __restrict__ rec, const float* dL_dop_eff,
                      float* dL_dopacity, const float* __restrict__ dL_dmean2D_abs,
                      float* __restrict__ grad_accum_abs) {
    extern __shared__ float bwd_smem[];
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int row_floats = vp.M * 3, stride = bwd_row_stride(row_floats);
    float* sh_rows = bwd_smem;                              // [kBwdBlock][stride] coefficients in
    float* dsh_rows = bwd_smem + kBwdBlock * stride;        // [kBwdBlock][stride] gradients out
    uint8_t* vis = reinterpret_cast<uint8_t*>(bwd_smem + 2 * kBwdBlock * stride);
    const int block_base = blockIdx.x * kBwdBlock;
    const int rows_here = min(kBwdBlock, vp.P - block_base);
    const bool visible = idx < vp.P && radii[idx] > 0;
    if (shs != nullptr) {
        vis[threadIdx.x] = visible ? 1 : 0;
        const float* src = shs + (size_t)block_base * row_floats;
        if ((row_floats & 3) == 0 && (reinterpret_cast<uintptr_t>(shs) & 15) == 0) {
            const int q_per_row = row_floats >> 2;
            for (int i = threadIdx.x; i < rows_here * q_per_row; i += kBwdBlock) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(src) + i);
                float* d = sh_rows + (i / q_per_row) * stride + (i % q_per_row) * 4;
                d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
            }
        } else {
            for (int i = threadIdx.x; i < rows_here * row_floats; i += kBwdBlock)
                sh_rows[(i / row_floats) * stride + (i % row_floats)] = __ldg(src + i);
        }
        // gradient rows start as zeros: degrees above the active one are not written by the owner thread
        for (int i = threadIdx.x; i < kBwdBlock * stride; i += kBwdBlock) dsh_rows[i] = 0.f;
        __syncthreads();
    }
    float cg[kCamTerms];  // CAM: this Gaussian's camera terms (slots above), 0 for a culled one
    if constexpr (CAM) {
#pragma unroll
        for (int j = 0; j < kCamTerms; j++) cg[j] = 0.f;
    }
    if (visible) {
    if (ACCUM && grad_accum != nullptr) {
        const float ux = dL_dmean2D[3 * idx], uy = dL_dmean2D[3 * idx + 1];
        grad_accum[idx] += sqrtf(ux * ux + uy * uy);
        vis_count[idx] += 1.0f;
        if constexpr (ABS) {
            const float ax = dL_dmean2D_abs[3 * idx], ay = dL_dmean2D_abs[3 * idx + 1];
            grad_accum_abs[idx] += sqrtf(ax * ax + ay * ay);
        }
    }
    const float* vm = vp.viewmatrix;
    const float* proj = vp.projmatrix;
    const float mx = means3D[3 * idx], my = means3D[3 * idx + 1], mz = means3D[3 * idx + 2];

    // ---- conic -> cov2D -> cov3D / mean (reference backward.cu:144-274)
    float cv[6];
#pragma unroll
    for (int i = 0; i < 6; i++) cv[i] = cov3D[6 * idx + i];
    const Cov2D c2 = project_cov(F3{mx, my, mz}, vm, vp.focal_x, vp.focal_y, vp.tan_fovx, vp.tan_fovy, cv);
    const float limx = 1.3f * vp.tan_fovx, limy = 1.3f * vp.tan_fovy;
    const float x_grad_mul = (c2.txtz < -limx || c2.txtz > limx) ? 0.f : 1.f;
    const float y_grad_mul = (c2.tytz < -limy || c2.tytz > limy) ? 0.f : 1.f;
    const float a = c2.a, b = c2.b, c = c2.c;
    const float dLcx = dL_dconic[4 * idx], dLcy = dL_dconic[4 * idx + 1], dLcz = dL_dconic[4 * idx + 3];
    const float denom = a * c - b * b;
    const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
    float dL_da = 0, dL_db = 0, dL_dc = 0;
    const float T00 = c2.T00, T01 = c2.T01, T02 = c2.T02, T10 = c2.T10, T11 = c2.T11, T12 = c2.T12;
    // AA: h = op_eff g / 2 where rho is not clamped.  Where it is (det0 / det <= kAaMinRatio, a degenerate undilated
    // covariance among them: det0 = 0 makes 1 / det0 infinite), rho is constant and nothing is added
    float aa_h = 0.f, det0 = 0.f;
    bool aa_terms = false;
    if constexpr (AA) {
        const float g = dL_dop_eff[idx];
        det0 = aa_det0(c2.a0, b, c2.c0);
        const float ratio = det0 / denom;
        put<ACCUM>(dL_dopacity + idx, sqrtf(fmaxf(kAaMinRatio, ratio)) * g);
        aa_terms = ratio > kAaMinRatio;
        if (aa_terms) aa_h = 0.5f * rec[idx].op * g;
    }
    float dcov[6];
    if (denom2inv != 0) {
        dL_da = denom2inv * (-c * c * dLcx + 2 * b * c * dLcy + (denom - a * c) * dLcz);
        dL_dc = denom2inv * (-a * a * dLcz + 2 * a * b * dLcy + (denom - a * c) * dLcx);
        dL_db = denom2inv * 2 * (b * c * dLcx - (denom + 2 * b * b) * dLcy + a * b * dLcz);
        if (AA && aa_terms) {
            // d log rho = (d det0 / det0 - d det / det) / 2, det0 = (a - 0.3)(c - 0.3) - b^2, det = a c - b^2
            dL_da += aa_h * (c2.c0 / det0 - c / denom);
            dL_dc += aa_h * (c2.a0 / det0 - a / denom);
            dL_db += 2.f * aa_h * b * (1.f / denom - 1.f / det0);
        }
        dcov[0] = (T00 * T00 * dL_da + T00 * T10 * dL_db + T10 * T10 * dL_dc);
        dcov[3] = (T01 * T01 * dL_da + T01 * T11 * dL_db + T11 * T11 * dL_dc);
        dcov[5] = (T02 * T02 * dL_da + T02 * T12 * dL_db + T12 * T12 * dL_dc);
        dcov[1] = 2 * T00 * T01 * dL_da + (T00 * T11 + T01 * T10) * dL_db + 2 * T10 * T11 * dL_dc;
        dcov[2] = 2 * T00 * T02 * dL_da + (T00 * T12 + T02 * T10) * dL_db + 2 * T10 * T12 * dL_dc;
        dcov[4] = 2 * T02 * T01 * dL_da + (T01 * T12 + T02 * T11) * dL_db + 2 * T11 * T12 * dL_dc;
    } else {
#pragma unroll
        for (int i = 0; i < 6; i++) dcov[i] = 0;
    }
#pragma unroll
    for (int i = 0; i < 6; i++) put<ACCUM>(dL_dcov3D + 6 * idx + i, dcov[i]);

    // Vrk rows (symmetric): V0 = (cv0,cv1,cv2), V1 = (cv1,cv3,cv4), V2 = (cv2,cv4,cv5)
    const float T0V0 = T00 * cv[0] + T01 * cv[1] + T02 * cv[2];
    const float T0V1 = T00 * cv[1] + T01 * cv[3] + T02 * cv[4];
    const float T0V2 = T00 * cv[2] + T01 * cv[4] + T02 * cv[5];
    const float T1V0 = T10 * cv[0] + T11 * cv[1] + T12 * cv[2];
    const float T1V1 = T10 * cv[1] + T11 * cv[3] + T12 * cv[4];
    const float T1V2 = T10 * cv[2] + T11 * cv[4] + T12 * cv[5];
    const float dL_dT00 = 2 * T0V0 * dL_da + T1V0 * dL_db;
    const float dL_dT01 = 2 * T0V1 * dL_da + T1V1 * dL_db;
    const float dL_dT02 = 2 * T0V2 * dL_da + T1V2 * dL_db;
    const float dL_dT10 = 2 * T1V0 * dL_dc + T0V0 * dL_db;
    const float dL_dT11 = 2 * T1V1 * dL_dc + T0V1 * dL_db;
    const float dL_dT12 = 2 * T1V2 * dL_dc + T0V2 * dL_db;
    // W columns: W[0] = (vm0, vm4, vm8), W[1] = (vm1, vm5, vm9), W[2] = (vm2, vm6, vm10)
    const float dL_dJ00 = vm[0] * dL_dT00 + vm[4] * dL_dT01 + vm[8] * dL_dT02;
    const float dL_dJ02 = vm[2] * dL_dT00 + vm[6] * dL_dT01 + vm[10] * dL_dT02;
    const float dL_dJ11 = vm[1] * dL_dT10 + vm[5] * dL_dT11 + vm[9] * dL_dT12;
    const float dL_dJ12 = vm[2] * dL_dT10 + vm[6] * dL_dT11 + vm[10] * dL_dT12;
    const float tz = 1.f / c2.tz;
    const float tz2 = tz * tz;
    const float tz3 = tz2 * tz;
    const float h_x = vp.focal_x, h_y = vp.focal_y;
    const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
    const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
    const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * c2.tx) * tz3 * dL_dJ02 +
                         (2 * h_y * c2.ty) * tz3 * dL_dJ12;
    // transformVec4x3Transpose
    float gx = vm[0] * dL_dtx + vm[1] * dL_dty + vm[2] * dL_dtz;
    float gy = vm[4] * dL_dtx + vm[5] * dL_dty + vm[6] * dL_dtz;
    float gz = vm[8] * dL_dtx + vm[9] * dL_dty + vm[10] * dL_dtz;
    if constexpr (CAM) {
        // t_r = xf(vm, r, p) gives dL/dvm[4k + r] = dL/dt_r p_k; T.c[a][k] = sum_r vm[4k + r] J.c[a][r] gives the W term
        // (J.c[0] = (fx/tz, 0, -fx tx/tz^2), J.c[1] = (0, fy/tz, -fy ty/tz^2), J.c[2] = 0)
        const float p[4] = {mx, my, mz, 1.f};
        float dT0[3] = {dL_dT00, dL_dT01, dL_dT02}, dT1[3] = {dL_dT10, dL_dT11, dL_dT12};
        float gtx = dL_dtx, gty = dL_dty, gtz = dL_dtz;
        float fx = h_x, fy = h_y, itz = tz, itz2 = tz2, ctx = c2.tx, cty = c2.ty;
        if constexpr (AA) {
            // as for the campos term below: the camera terms read opaque copies, so that a second use of these values
            // cannot change how the compiler contracts the other outputs of the antialiased kernels
            asm("" : "+f"(dT0[0]), "+f"(dT0[1]), "+f"(dT0[2]), "+f"(dT1[0]), "+f"(dT1[1]), "+f"(dT1[2]));
            asm("" : "+f"(gtx), "+f"(gty), "+f"(gtz), "+f"(fx), "+f"(fy), "+f"(itz), "+f"(itz2), "+f"(ctx), "+f"(cty));
        }
        const float J00 = fx * itz, J11 = fy * itz, J02 = -fx * ctx * itz2, J12 = -fy * cty * itz2;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            cg[3 * k] = gtx * p[k];
            cg[3 * k + 1] = gty * p[k];
            cg[3 * k + 2] = gtz * p[k];
            if (k < 3) {
                cg[3 * k] += dT0[k] * J00;
                cg[3 * k + 1] += dT1[k] * J11;
                cg[3 * k + 2] += dT0[k] * J02 + dT1[k] * J12;
            }
        }
    }

    // ---- screen-space mean and depth (reference backward.cu:372-395)
    {
        const float hw = proj[3] * mx + proj[7] * my + proj[11] * mz + proj[15];
        const float m_w = 1.0f / (hw + 0.0000001f);
        const float mul1 = (proj[0] * mx + proj[4] * my + proj[8] * mz + proj[12]) * m_w * m_w;
        const float mul2 = (proj[1] * mx + proj[5] * my + proj[9] * mz + proj[13]) * m_w * m_w;
        const float d2x = dL_dmean2D[3 * idx], d2y = dL_dmean2D[3 * idx + 1];
        float ax = (proj[0] * m_w - proj[3] * mul1) * d2x + (proj[1] * m_w - proj[3] * mul2) * d2y;
        float ay = (proj[4] * m_w - proj[7] * mul1) * d2x + (proj[5] * m_w - proj[7] * mul2) * d2y;
        float az = (proj[8] * m_w - proj[11] * mul1) * d2x + (proj[9] * m_w - proj[11] * mul2) * d2y;
        const float dldz = dL_dz[idx];
        ax += dldz * vm[2];
        ay += dldz * vm[6];
        az += dldz * vm[10];
        gx += ax; gy += ay; gz += az;
        if constexpr (CAM) {
            // proj = (h_0, h_1) m_w with h_r = xf(pm, r, p): dL/dh_0 = m_w d2x, dL/dh_1 = m_w d2y,
            // dL/dh_3 = -(mul1 d2x + mul2 d2y); depth = xf(vm, 2, p)
            const float p[4] = {mx, my, mz, 1.f};
            float w = m_w, gx2 = d2x, gy2 = d2y, u1 = mul1, u2 = mul2, gdz = dldz;
            if constexpr (AA) asm("" : "+f"(w), "+f"(gx2), "+f"(gy2), "+f"(u1), "+f"(u2), "+f"(gdz));  // as above
            const float gh[3] = {w * gx2, w * gy2, -(u1 * gx2 + u2 * gy2)};
#pragma unroll
            for (int k = 0; k < 4; k++) {
                cg[3 * k + 2] += gdz * p[k];
#pragma unroll
                for (int i = 0; i < 3; i++) cg[12 + 3 * k + i] = gh[i] * p[k];
            }
        }
    }

    // ---- SH backward (reference backward.cu:20-139)
    if (shs != nullptr) {
        const float* sh = sh_rows + threadIdx.x * stride;
        float* dsh = dsh_rows + threadIdx.x * stride;
        const float* cam = vp.cam_pos;
        F3 dir_orig = {mx - cam[0], my - cam[1], mz - cam[2]};
        const float inv_len = 1.0f / sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
        const float x = dir_orig.x * inv_len, y = dir_orig.y * inv_len, z = dir_orig.z * inv_len;
        const uint8_t cb = clamped[idx];
        float dRGB[3];
        dRGB[0] = (cb & 1) ? 0.f : dL_dcolor[3 * idx];
        dRGB[1] = (cb & 2) ? 0.f : dL_dcolor[3 * idx + 1];
        dRGB[2] = (cb & 4) ? 0.f : dL_dcolor[3 * idx + 2];
        F3 dd, dm;
        if constexpr (AA) {
            dm = sh_backward_out_of_line(vp.D, sh, dsh, dRGB[0], dRGB[1], dRGB[2], dir_orig, &dd);
        } else {
            dd = sh_dir_grad(vp.D, sh, dsh, dRGB, x, y, z);
            dm = dnormvdv3(dir_orig, dd);
        }
        gx += dm.x; gy += dm.y; gz += dm.z;
        if constexpr (CAM) {
            // dir_orig = p - campos: dL/dcampos = -dm.  dm is recomputed from opaque copies of its inputs rather than
            // read: a second use of dm's products would change how the compiler contracts `gx += dm.x` into FMAs, and
            // so the bits of dL_dmean3D, which must equal those of the CAM = false kernel.
            if constexpr (AA) {  // dm comes from the out-of-line call: a second use cannot change its bits
                cg[24] = -dm.x; cg[25] = -dm.y; cg[26] = -dm.z;
            } else {
                F3 v = dir_orig, dv = dd;
                asm("" : "+f"(v.x), "+f"(v.y), "+f"(v.z), "+f"(dv.x), "+f"(dv.y), "+f"(dv.z));
                const F3 dmc = dnormvdv3(v, dv);
                cg[24] = -dmc.x; cg[25] = -dmc.y; cg[26] = -dmc.z;
            }
        }
    }
    put<ACCUM>(dL_dmean3D + 3 * idx, gx);
    put<ACCUM>(dL_dmean3D + 3 * idx + 1, gy);
    put<ACCUM>(dL_dmean3D + 3 * idx + 2, gz);

    // ---- cov3D -> scale / rotation (reference backward.cu:278-341)
    if (scales != nullptr) {
        const float r = rotations[4 * idx], x = rotations[4 * idx + 1], y = rotations[4 * idx + 2],
                    z = rotations[4 * idx + 3];
        // R in GLM column-major: R[c][r]
        const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                               {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                               {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
        const float s[3] = {vp.scale_modifier * scales[3 * idx], vp.scale_modifier * scales[3 * idx + 1],
                            vp.scale_modifier * scales[3 * idx + 2]};
        // M = S * R  ->  M[c][r] = s[r] * R[c][r]
        float M[3][3];
#pragma unroll
        for (int cc = 0; cc < 3; cc++)
#pragma unroll
            for (int rr = 0; rr < 3; rr++) M[cc][rr] = s[rr] * R[cc][rr];
        // dL_dSigma (symmetric, column-major irrelevant)
        const float S[3][3] = {{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]},
                               {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]},
                               {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}};
        // dL_dM = 2 * M * dL_dSigma : (A*B)[c][r] = sum_k A[k][r] * B[c][k]
        float dM[3][3];
#pragma unroll
        for (int cc = 0; cc < 3; cc++)
#pragma unroll
            for (int rr = 0; rr < 3; rr++)
                dM[cc][rr] = 2.0f * (M[0][rr] * S[cc][0] + M[1][rr] * S[cc][1] + M[2][rr] * S[cc][2]);
        // Rt[c][r] = R[r][c]; dL_dMt[c][r] = dM[r][c]; dL_dscale_k = dot(Rt[k], dL_dMt[k])
        float dMt[3][3];
#pragma unroll
        for (int cc = 0; cc < 3; cc++)
#pragma unroll
            for (int rr = 0; rr < 3; rr++) dMt[cc][rr] = dM[rr][cc];
#pragma unroll
        for (int k = 0; k < 3; k++)
            put<ACCUM>(dL_dscale + 3 * idx + k, R[0][k] * dMt[k][0] + R[1][k] * dMt[k][1] + R[2][k] * dMt[k][2]);
#pragma unroll
        for (int k = 0; k < 3; k++)
#pragma unroll
            for (int rr = 0; rr < 3; rr++) dMt[k][rr] *= s[k];
        float4 dq;
        dq.x = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
        dq.y = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) -
               4 * x * (dMt[2][2] + dMt[1][1]);
        dq.z = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) -
               4 * y * (dMt[2][2] + dMt[0][0]);
        dq.w = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) -
               4 * z * (dMt[1][1] + dMt[0][0]);
        if (ACCUM) {
            const float4 o = reinterpret_cast<float4*>(dL_drot)[idx];
            dq.x += o.x; dq.y += o.y; dq.z += o.z; dq.w += o.w;
        }
        reinterpret_cast<float4*>(dL_drot)[idx] = dq;
    }
    }  // visible
    if (shs != nullptr) {
        // coalesced write-out of the block's gradient rows (rows of culled Gaussians stay untouched: zero / unchanged)
        __syncthreads();
        float* dst = dL_dsh + (size_t)block_base * row_floats;
        if ((row_floats & 3) == 0 && (reinterpret_cast<uintptr_t>(dL_dsh) & 15) == 0) {
            const int q_per_row = row_floats >> 2;
            for (int i = threadIdx.x; i < rows_here * q_per_row; i += kBwdBlock) {
                const int row = i / q_per_row;
                if (!vis[row]) continue;
                const float* g = dsh_rows + row * stride + (i % q_per_row) * 4;
                float4 v = make_float4(g[0], g[1], g[2], g[3]);
                float4* o = reinterpret_cast<float4*>(dst) + i;
                if (ACCUM) {
                    const float4 old = *o;
                    v.x += old.x; v.y += old.y; v.z += old.z; v.w += old.w;
                }
                *o = v;
            }
        } else {
            for (int i = threadIdx.x; i < rows_here * row_floats; i += kBwdBlock) {
                const int row = i / row_floats;
                if (!vis[row]) continue;
                const float g = dsh_rows[row * stride + (i % row_floats)];
                dst[i] = ACCUM ? dst[i] + g : g;
            }
        }
    }
    if constexpr (CAM) {
        // fixed-order block reduction: float32 warp shuffles, then the four warp sums in float64 -> cam_part[block][27]
        __shared__ float cam_warp[kBwdBlock / 32][kCamTerms];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int j = 0; j < kCamTerms; j++) {
            float v = cg[j];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
            if (lane == 0) cam_warp[warp][j] = v;
        }
        __syncthreads();
        if (threadIdx.x < kCamTerms) {
            double s = 0.0;
#pragma unroll
            for (int w = 0; w < kBwdBlock / 32; w++) s += (double)cam_warp[w][threadIdx.x];
            cam_part[(size_t)blockIdx.x * kCamTerms + threadIdx.x] = s;
        }
    }
}

// dL_dcamera[cam_slot(j)] += the float64 sum of the blocks' partials of slot j (one CTA per slot; each thread sums a
// fixed stride of blocks in index order, then a fixed tree), rounded once to float32
constexpr int kCamSumThreads = 256;
__global__ void __launch_bounds__(kCamSumThreads)
camera_grad_sum_kernel(int blocks, const double* __restrict__ cam_part, float* __restrict__ dL_dcamera) {
    __shared__ double s[kCamSumThreads];
    const int j = blockIdx.x;
    double a = 0.0;
    for (int b = threadIdx.x; b < blocks; b += kCamSumThreads) a += cam_part[(size_t)b * kCamTerms + j];
    s[threadIdx.x] = a;
    __syncthreads();
#pragma unroll
    for (int w = kCamSumThreads / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) dL_dcamera[cam_slot(j)] += (float)s[0];
}

// -------------------------------------------------------------------------------- launchers
void launch_preprocess_fwd(const ViewParams& vp, const float* means3D, const float* scales,
                           const float* rotations, const float* opacities, const float* shs,
                           const float* cov3D_precomp, const float* colors_precomp, bool prefiltered,
                           int* radii, SplatRec* rec, float* cov3D, uint8_t* clamped,
                           uint32_t* tiles_touched, cudaStream_t s, bool antialiasing) {
    if (vp.P <= 0) return;
    constexpr int kFwdBlock = 128;
    const size_t smem = shs ? (size_t)kFwdBlock * bwd_row_stride(vp.M * 3) * sizeof(float) : 0;
    const auto kernel = antialiasing ? preprocess_fwd_kernel<true> : preprocess_fwd_kernel<false>;
    kernel<<<(vp.P + kFwdBlock - 1) / kFwdBlock, kFwdBlock, smem, s>>>(vp, means3D, scales, rotations, opacities, shs,
                                                                       cov3D_precomp, colors_precomp, prefiltered, radii,
                                                                       rec, cov3D, clamped, tiles_touched);
    g_launches++;
}

cudaError_t launch_preprocess_bwd(const ViewParams& vp, const float* means3D, const int* radii, const float* shs,
                                  const uint8_t* clamped, const float* scales, const float* rotations,
                                  const float* cov3D, const float* dL_dmean2D, const float* dL_dconic,
                                  float* dL_dmean3D, const float* dL_dcolor, float* dL_dcov3D, float* dL_dsh,
                                  float* dL_dscale, float* dL_drot, const float* dL_dz, cudaStream_t s, bool accumulate,
                                  float* grad_accum, float* denom, float* dL_dcamera, bool antialiasing,
                                  const SplatRec* rec, const float* dL_dop_eff, float* dL_dopacity,
                                  const float* dL_dmean2D_abs, float* grad_accum_abs) {
    if (vp.P <= 0) return cudaSuccess;
    using Kernel = decltype(&preprocess_bwd_kernel<false, false, false>);
    // [accumulate][camera][antialiasing]
    static const Kernel kernels[2][2][2] = {
        {{preprocess_bwd_kernel<false, false, false>, preprocess_bwd_kernel<false, false, true>},
         {preprocess_bwd_kernel<false, true, false>, preprocess_bwd_kernel<false, true, true>}},
        {{preprocess_bwd_kernel<true, false, false>, preprocess_bwd_kernel<true, false, true>},
         {preprocess_bwd_kernel<true, true, false>, preprocess_bwd_kernel<true, true, true>}}};
    // the accumulating backward with AbsGS's statistic: [camera][antialiasing]
    static const Kernel abs_kernels[2][2] = {
        {preprocess_bwd_kernel<true, false, false, true>, preprocess_bwd_kernel<true, false, true, true>},
        {preprocess_bwd_kernel<true, true, false, true>, preprocess_bwd_kernel<true, true, true, true>}};
    const size_t smem = shs ? (size_t)2 * kBwdBlock * bwd_row_stride(vp.M * 3) * sizeof(float) + kBwdBlock : 0;
    static std::atomic<int> attr_set{0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (smem > 48 * 1024 && !((attr_set.load() >> (dev & 31)) & 1)) {  // once per device; harmless if repeated
        for (const Kernel k : {kernels[0][0][0], kernels[0][0][1], kernels[0][1][0], kernels[0][1][1], kernels[1][0][0],
                               kernels[1][0][1], kernels[1][1][0], kernels[1][1][1], abs_kernels[0][0],
                               abs_kernels[0][1], abs_kernels[1][0], abs_kernels[1][1]})
            cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        attr_set.fetch_or(1 << (dev & 31));
    }
    const int grid = (vp.P + kBwdBlock - 1) / kBwdBlock;
    const bool cam = dL_dcamera != nullptr;
    // the camera gradient's block partials come from the device's default memory pool, stream-ordered like the launches
    double* part = nullptr;
    if (cam) {
        const cudaError_t e = cudaMallocAsync((void**)&part, (size_t)grid * kCamTerms * sizeof(double), s);
        if (e != cudaSuccess) return e;
    }
    const bool abs = accumulate && grad_accum && grad_accum_abs;
    (abs ? abs_kernels[cam][antialiasing] : kernels[accumulate][cam][antialiasing])<<<grid, kBwdBlock, smem, s>>>(
        vp, means3D, radii, shs, clamped, scales, rotations, cov3D, dL_dmean2D, dL_dconic, dL_dmean3D, dL_dcolor,
        dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dz, accumulate ? grad_accum : nullptr, accumulate ? denom : nullptr,
        part, rec, dL_dop_eff, dL_dopacity, abs ? dL_dmean2D_abs : nullptr, abs ? grad_accum_abs : nullptr);
    g_launches++;
    if (!cam) return cudaSuccess;  // a launch error is left for the caller's cudaGetLastError
    camera_grad_sum_kernel<<<kCamTerms, kCamSumThreads, 0, s>>>(grid, part, dL_dcamera);
    g_launches++;
    return cudaFreeAsync(part, s);
}

void launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                         cudaStream_t s) {
    if (P <= 0) return;
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, means3D, viewmatrix, present);
    g_launches++;
}

}  // namespace f3dgs
