// Adaptive density control: clone / split / prune with the Adam state carried along, and the opacity reset
// (reference scene/gaussian_model.py:350-434 densify_and_prune, :231-234 reset_opacity).
//
// The result is the order-preserving compaction of the virtual row list
//     [P originals | clones, in index order | split copy 0 of every split Gaussian | split copy 1]
// that drops the originals selected for split and every row that fails the prune test.  Per Gaussian i:
//   g = grad_accum / denom (NaN -> 0), smax = max over 3 of expf(raw_scaling), o = sigmoid(raw_opacity)
//   clone  g >= max_grad && smax <= dense_scale
//   split  g >= max_grad && smax >  dense_scale
//          (AbsGS, with grad_accum_abs: ga >= abs_grad && smax > dense_scale, ga = grad_accum_abs / denom, NaN -> 0)
//   prune  o < min_opacity || smax > max_world_scale   (each row with its own scaling; a child's is
//                                                        logf(expf(raw) * (1 / 1.6f)), the reference's log(s / (0.8 N)))
// Both split copies share scaling and opacity, so they are kept or pruned together.
//
// Pipeline (stream-ordered):
//   1. classify_kernel  one thread per Gaussian: int4 {original kept, clone kept, child kept, split} (row P: zeros)
//   2. cub::DeviceScan::ExclusiveScan (in place, P + 1 items) -> every output position; row P holds the totals
//      {A, B, Cc, Ns}, copied to the caller's counts[4]
//   3. apply_kernel     one launch over a flat work list of every (tensor, element) pair of the 21 source tensors
//      (7 raw fields, exp_avg, exp_avg_sq): each element is read once and written to its original row, its clone row
//      and its two child rows (moments: zeros for the new rows).  Child xyz = R(q) (z * std) + parent xyz with z the
//      caller's normals, child scaling as above.  Every new row is written exactly once; no atomics, so the result is
//      bitwise reproducible.
// A prune from the caller's mask (f3dgs_prune_plan) replaces step 1 by prune_classify_kernel, flags {keep != 0, 0, 0, 0};
// the scan and apply_kernel are the same, with totals {A, 0, 0, 0} and no normals.
#include <cub/cub.cuh>

#include <cmath>

#include "kernels.h"

namespace f3dgs {

namespace {

struct Add4 {
    __device__ __forceinline__ int4 operator()(const int4& a, const int4& b) const {
        return make_int4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
};

cudaError_t scan_bytes(int P, size_t* bytes) {
    *bytes = 0;
    return cub::DeviceScan::ExclusiveScan(nullptr, *bytes, (int4*)nullptr, (int4*)nullptr, Add4(), make_int4(0, 0, 0, 0),
                                          P + 1);
}

// step 2 after a classify launch: the flags scanned in place, their totals copied to counts
cudaError_t scan_flags(int P, char* scratch, int32_t* counts, cudaStream_t s) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t sb = 0;
    if ((e = scan_bytes(P, &sb)) != cudaSuccess) return e;
    int4* flags = reinterpret_cast<int4*>(scratch);
    if ((e = cub::DeviceScan::ExclusiveScan(scratch + densify_scratch_fixed_bytes(P), sb, flags, flags, Add4(),
                                            make_int4(0, 0, 0, 0), P + 1, s)) != cudaSuccess)
        return e;
    return cudaMemcpyAsync(counts, flags + P, 4 * sizeof(int32_t), cudaMemcpyDeviceToDevice, s);
}

// torch's max over a dimension: NaN propagates
__device__ __forceinline__ float max3_nan(float a, float b, float c) {
    float m = a;
    m = (m != m || m >= b) ? m : b;
    m = (m != m || m >= c) ? m : c;
    return m;
}

// the split child's raw scaling: torch's log(exp(s) / (0.8 * N)) on CUDA multiplies by the fp32 reciprocal
__device__ __forceinline__ float child_scaling(float raw, float split_inv) { return logf(expf(raw) * split_inv); }

struct ClassifyArgs {
    int P;
    const float *grad_accum, *denom, *raw_opacity, *raw_scaling;
    float max_grad, dense_scale, min_opacity, max_world_scale, split_inv;
    int4* flags;
    const float* grad_accum_abs;  // ABS
    float abs_grad;               // ABS
};

template <bool ABS = false>
__global__ void __launch_bounds__(256) classify_kernel(const __grid_constant__ ClassifyArgs a) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i > a.P) return;
    if (i == a.P) {
        a.flags[i] = make_int4(0, 0, 0, 0);
        return;
    }
    float g = a.grad_accum[i] / a.denom[i];
    if (g != g) g = 0.0f;
    const float r0 = a.raw_scaling[3 * i], r1 = a.raw_scaling[3 * i + 1], r2 = a.raw_scaling[3 * i + 2];
    const float smax = max3_nan(expf(r0), expf(r1), expf(r2));
    const float o = 1.0f / (1.0f + expf(-a.raw_opacity[i]));  // torch.sigmoid
    const bool transparent = o < a.min_opacity;
    const bool sel = g >= a.max_grad;
    bool split_sel = sel;
    if constexpr (ABS) {
        float ga = a.grad_accum_abs[i] / a.denom[i];
        if (ga != ga) ga = 0.0f;
        split_sel = ga >= a.abs_grad;
    }
    const bool clone = sel && smax <= a.dense_scale, split = split_sel && smax > a.dense_scale;
    const bool prune = transparent || smax > a.max_world_scale;  // the clone shares the original's scaling
    int child = 0;
    if (split) {
        const float cmax = max3_nan(expf(child_scaling(r0, a.split_inv)), expf(child_scaling(r1, a.split_inv)),
                                    expf(child_scaling(r2, a.split_inv)));
        child = !(transparent || cmax > a.max_world_scale);
    }
    a.flags[i] = make_int4(!split && !prune, clone && !prune, child, split);
}

__global__ void __launch_bounds__(256) prune_classify_kernel(int P, const uint8_t* __restrict__ keep, int4* flags) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i > P) return;
    flags[i] = make_int4(i < P && keep[i] != 0, 0, 0, 0);
}

// One segment per (group, field): group 0 the raw parameters, 1 exp_avg, 2 exp_avg_sq; fields in
// f3dgs_gaussian_fields order.  A block covers kChunk consecutive elements of one segment.
constexpr int kSegs = 21, kThreads = 256, kPerThread = 8, kChunk = kThreads * kPerThread;
constexpr int kFieldXyz = 0, kFieldScaling = 4;

struct ApplyArgs {
    const float* src[kSegs];
    float* dst[kSegs];
    int width[kSegs];                     // floats per row
    unsigned long long block_end[kSegs];  // exclusive prefix of the segments' block counts
    const int4* scan;                     // [P + 1]: exclusive scan of the classify flags, totals at P
    const float *raw_scaling, *raw_rotation, *normals;
    int A, B, Cc, Ns;
    float split_inv;
};

// xyz of split copy r of Gaussian `row`, component `col`: R(q) (z * std) + parent, q = r / sqrt(sum r^2)
// (utils/general_utils.py build_rotation, w x y z).  R and z * std are rounded step by step as the reference's
// elementwise tensor ops round them (no contraction); only the 3-term dot product has an order of its own.
__device__ __forceinline__ float sq_sum(float a, float b) { return __fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)); }
__device__ __forceinline__ float diag(float a, float b) { return __fsub_rn(1.f, 2.f * sq_sum(a, b)); }
__device__ __forceinline__ float off(float a, float b, float c, float d, float sign) {
    return 2.f * __fadd_rn(__fmul_rn(a, b), sign * __fmul_rn(c, d));
}

__device__ __forceinline__ float child_xyz(const ApplyArgs& a, size_t row, int col, float parent, int zrow) {
    const float4 r = reinterpret_cast<const float4*>(a.raw_rotation)[row];
    const float n = sqrtf(__fadd_rn(__fadd_rn(sq_sum(r.x, r.y), __fmul_rn(r.z, r.z)), __fmul_rn(r.w, r.w)));
    const float w = r.x / n, x = r.y / n, y = r.z / n, z = r.w / n;
    float R0, R1, R2;
    if (col == 0) {
        R0 = diag(y, z); R1 = off(x, y, w, z, -1.f); R2 = off(x, z, w, y, 1.f);
    } else if (col == 1) {
        R0 = off(x, y, w, z, 1.f); R1 = diag(x, z); R2 = off(y, z, w, x, -1.f);
    } else {
        R0 = off(x, z, w, y, -1.f); R1 = off(y, z, w, x, 1.f); R2 = diag(x, y);
    }
    const float* s = a.raw_scaling + 3 * row;
    const float* nz = a.normals + 3 * (size_t)zrow;
    const float v0 = __fmul_rn(nz[0], expf(s[0])), v1 = __fmul_rn(nz[1], expf(s[1])), v2 = __fmul_rn(nz[2], expf(s[2]));
    return __fadd_rn(__fmaf_rn(R2, v2, __fmaf_rn(R1, v1, __fmul_rn(R0, v0))), parent);
}

__global__ void __launch_bounds__(kThreads) apply_kernel(const __grid_constant__ ApplyArgs a, int P) {
    // a caller whose counts disagree with the plan's would size the outputs wrongly: write nothing
    const int4 tot = a.scan[P];
    if (tot.x != a.A || tot.y != a.B || tot.z != a.Cc || tot.w != a.Ns) return;
    int seg = 0;
    while (blockIdx.x >= a.block_end[seg]) seg++;
    const unsigned long long first = seg ? a.block_end[seg - 1] : 0ull;
    const int w = a.width[seg], group = seg / 7, field = seg % 7;
    const float* __restrict__ src = a.src[seg];
    float* __restrict__ dst = a.dst[seg];
    const size_t n = (size_t)P * w;
    size_t e = (size_t)(blockIdx.x - first) * kChunk + threadIdx.x;
    size_t row = e / w;
    int col = (int)(e - row * w);
    const int dq = kThreads / w, dr = kThreads % w;
    for (int k = 0; k < kPerThread && e < n; k++, e += kThreads) {
        const int4 s0 = a.scan[row], s1 = a.scan[row + 1];
        const bool keep = s1.x != s0.x, clone = s1.y != s0.y, child = s1.z != s0.z;
        if (keep | clone | child) {
            const float v = src[e];
            if (keep) dst[(size_t)s0.x * w + col] = v;
            const float vn = group ? 0.0f : v;  // the moments of new rows start at zero
            if (clone) dst[(size_t)(a.A + s0.y) * w + col] = vn;
            if (child) {
                float c0 = vn, c1 = vn;
                if (group == 0 && field == kFieldScaling) {
                    c0 = c1 = child_scaling(v, a.split_inv);
                } else if (group == 0 && field == kFieldXyz) {
                    c0 = child_xyz(a, row, col, v, s0.w);
                    c1 = child_xyz(a, row, col, v, a.Ns + s0.w);
                }
                const size_t r0 = (size_t)(a.A + a.B) + s0.z;
                dst[r0 * w + col] = c0;
                dst[(r0 + a.Cc) * w + col] = c1;
            }
        }
        col += dr;
        row += dq;
        if (col >= w) {
            col -= w;
            row++;
        }
    }
}

__global__ void __launch_bounds__(256) reset_opacity_kernel(int P, float* __restrict__ raw, float* __restrict__ m,
                                                            float* __restrict__ v, float ceiling) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float o = 1.0f / (1.0f + expf(-raw[i]));  // torch.sigmoid
    const float x = (o != o) ? o : fminf(o, ceiling);  // torch.minimum: NaN propagates
    raw[i] = logf(x / (1.0f - x));                     // inverse_sigmoid
    m[i] = 0.0f;
    v[i] = 0.0f;
}

}  // namespace

cudaError_t densify_scratch_bytes(int P, size_t* bytes) {
    *bytes = 0;
    if (P <= 0) return cudaSuccess;
    size_t sb = 0;
    const cudaError_t e = scan_bytes(P, &sb);
    if (e != cudaSuccess) return e;
    *bytes = densify_scratch_fixed_bytes(P) + align_up(sb);
    return cudaSuccess;
}

size_t densify_scratch_fixed_bytes(int P) { return P > 0 ? align_up(((size_t)P + 1) * sizeof(int4)) : 0; }

float densify_split_inv() { return 1.0f / (float)(0.8 * 2); }  // as torch: opmath(1) / float(scalar), on the host

cudaError_t launch_densify_plan(int P, const float* grad_accum, const float* denom, const float* raw_opacity,
                                const float* raw_scaling, float max_grad, float dense_scale, float min_opacity,
                                float max_world_scale, char* scratch, int32_t* counts, cudaStream_t s,
                                const float* grad_accum_abs, float abs_grad) {
    if (P == 0) return cudaMemsetAsync(counts, 0, 4 * sizeof(int32_t), s);
    int4* flags = reinterpret_cast<int4*>(scratch);
    ClassifyArgs c{};
    c.P = P; c.grad_accum = grad_accum; c.denom = denom; c.raw_opacity = raw_opacity; c.raw_scaling = raw_scaling;
    c.max_grad = max_grad; c.dense_scale = dense_scale; c.min_opacity = min_opacity; c.max_world_scale = max_world_scale;
    c.split_inv = densify_split_inv(); c.flags = flags;
    c.grad_accum_abs = grad_accum_abs; c.abs_grad = abs_grad;
    if (grad_accum_abs)
        classify_kernel<true><<<blocks_for((long long)P + 1), 256, 0, s>>>(c);
    else
        classify_kernel<<<blocks_for((long long)P + 1), 256, 0, s>>>(c);
    g_launches++;
    return scan_flags(P, scratch, counts, s);
}

cudaError_t launch_prune_plan(int P, const uint8_t* keep, char* scratch, int32_t* counts, cudaStream_t s) {
    if (P == 0) return cudaMemsetAsync(counts, 0, 4 * sizeof(int32_t), s);
    prune_classify_kernel<<<blocks_for((long long)P + 1), 256, 0, s>>>(P, keep, reinterpret_cast<int4*>(scratch));
    g_launches++;
    return scan_flags(P, scratch, counts, s);
}

cudaError_t launch_densify_apply(int P, int M, int C, const char* scratch, const int32_t counts[4], const float* normals,
                                 const float* const src[21], float* const dst[21], cudaStream_t s) {
    const int A = counts[0], B = counts[1], Cc = counts[2], Ns = counts[3];
    if (P == 0 || A + B + 2 * (long long)Cc == 0) return cudaSuccess;
    const int width[7] = {3, 3, 3 * (M - 1), 1, 3, 4, C};
    ApplyArgs a;
    unsigned long long blocks = 0;
    for (int k = 0; k < kSegs; k++) {
        a.src[k] = src[k];
        a.dst[k] = dst[k];
        a.width[k] = width[k % 7];
        blocks += ((unsigned long long)P * width[k % 7] + kChunk - 1) / kChunk;
        a.block_end[k] = blocks;
    }
    a.scan = reinterpret_cast<const int4*>(scratch);
    a.raw_scaling = src[kFieldScaling];
    a.raw_rotation = src[5];
    a.normals = normals;
    a.A = A; a.B = B; a.Cc = Cc; a.Ns = Ns;
    a.split_inv = densify_split_inv();
    if (blocks > 0x7fffffffull) return cudaErrorInvalidConfiguration;
    apply_kernel<<<(unsigned)blocks, kThreads, 0, s>>>(a, P);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_reset_opacity(int P, float* raw_opacity, float* exp_avg, float* exp_avg_sq, float ceiling,
                                 cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    reset_opacity_kernel<<<blocks_for(P), 256, 0, s>>>(P, raw_opacity, exp_avg, exp_avg_sq, ceiling);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace f3dgs
