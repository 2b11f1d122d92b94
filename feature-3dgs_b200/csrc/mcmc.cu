// Fixed-budget densification: the relocation and growth of 3DGS-MCMC (Kheradmand et al., "3D Gaussian Splatting as
// Markov Chain Monte Carlo", NeurIPS 2024; the official code's relocate_gs / add_new_gs, gsplat's MCMCStrategy) and
// its position noise, with the Adam state carried along.
//
// Relocation rule.  A source Gaussian of opacity o and scales s drawn c >= 1 times ends as N = min(c + 1, 51) identical
// Gaussians (itself plus one copy per draw; 51 is gsplat's n_max), each with
//   o' = 1 - (1 - o)^(1/N) = -expm1(log1p(-o) / N)
//   s' = s * o / D(o', N),   D(x, N) = sum_{j=1..N} C(N,j) (-1)^(j-1) x^j / sqrt(j)
// D is the official kernel's double loop sum_{i=1..N} sum_{k<i} C(i-1,k) (-1)^k x^(k+1) / sqrt(k+1) summed in closed
// form (hockey-stick identity).  Both are evaluated in double from the float o = sigmoid(raw) and s = exp(raw), o' is
// clamped to [min_opacity, 1 - FLT_EPSILON] (s' uses the unclamped o'), and the raw fields logit(o') and log(s') are
// rounded to float once.  The official float32 loop with powf loses up to 8e-4 of o' at N = 51 to cancellation.
//
// Pipelines (stream-ordered, one scratch):
//   plan      classify (dead = o <= min_opacity), cub exclusive sum, scatter: index = [dead ascending | alive
//             ascending], alive_opacity in the alive order, n_dead on the device.
//   relocate  count the draws per source (integer atomics; an index outside [0, P) raises a device flag and every
//             later kernel writes nothing), then (o', s') per draw from the old values, then one pass over every
//             (draw, element): the dead row takes its source's raw fields with (o', s'), the source takes (o', s'), its
//             moments are zeroed; an optional float16 feature copy takes the dead row's features.  The dead row's
//             moments are left as they were: the official code and gsplat do the same (they reset the sources' state
//             only), so a relocated row starts from the moments of the Gaussian that died there.
//   add       count the draws per source, (o', s') per draw, exclusive sum -> each source's list of draws, then one
//             pass over every old element: it is read at most once and written to its own row and to the rows P + j
//             of every draw j of its row; drawn rows get (o', s') and zero moments, new rows zero moments.  No float
//             atomics: all copies of a source are identical, so the order inside a list does not change the output.
//   noise     one thread per Gaussian: xyz += R diag(s^2) R^T (eps * g * scale), g = 1 / (1 + exp(-100 ((1 - o) -
//             0.995))), in double, rounded once.
// Every kernel is bitwise reproducible for equal inputs.
#include <cub/cub.cuh>

#include <cfloat>
#include <cmath>

#include "kernels.h"

namespace f3dgs {

namespace {

constexpr int kNMax = 51;
constexpr int kFieldOpacity = 3, kFieldScaling = 4, kFieldFeature = 6;

cudaError_t scan_bytes(int P, size_t* bytes) {
    *bytes = 0;
    return cub::DeviceScan::ExclusiveSum(nullptr, *bytes, (int*)nullptr, (int*)nullptr, P + 1);
}

// scratch layout: [err flag | int[P + 1] flags / counts / offsets | float4 values[P] per draw | cursor[P] | list[P] |
// cub temp]
struct Scratch {
    int* err;
    int* counts;
    float4* per_draw;
    int *cursor, *list;
    char* cub;
    explicit Scratch(int P, char* base) {
        err = reinterpret_cast<int*>(base);
        counts = reinterpret_cast<int*>(base + 256);
        char* b = base + 256 + align_up(((size_t)P + 1) * 4);
        per_draw = reinterpret_cast<float4*>(b);
        cursor = reinterpret_cast<int*>(b + (size_t)P * 16);
        list = cursor + P;
        cub = b + align_up((size_t)P * 24);
    }
};

__device__ __forceinline__ float sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }  // torch.sigmoid

// o' (unclamped) and o / D(o', N) in double
__device__ __forceinline__ void relocation(float o, int N, double& op, double& ratio) {
    const double od = o;
    op = -expm1(log1p(-od) / N);
    double c = 1.0, p = 1.0, D = 0.0;
    for (int j = 1; j <= N; j++) {
        c = c * (N - j + 1) / j;  // C(N, j)
        p *= op;
        const double t = c * p / sqrt((double)j);
        D += (j & 1) ? t : -t;
    }
    ratio = od / D;
}

__device__ __forceinline__ float raw_opacity_of(double op, float min_opacity) {
    const double x = fmin(fmax(op, (double)min_opacity), 1.0 - (double)FLT_EPSILON);
    return (float)log(x / (1.0 - x));
}

__device__ __forceinline__ float raw_scaling_of(float raw_s, double ratio) {
    return (float)log((double)expf(raw_s) * ratio);
}

__device__ __forceinline__ int copies(int count) { return min(count + 1, kNMax); }

// ---- plan
__global__ void __launch_bounds__(256) classify_kernel(int P, const float* __restrict__ raw_opacity, float min_opacity,
                                                       int* __restrict__ flags) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i > P) return;
    flags[i] = i < P && sigmoid(raw_opacity[i]) <= min_opacity;
}

__global__ void __launch_bounds__(256) scatter_kernel(int P, const float* __restrict__ raw_opacity, float min_opacity,
                                                      const int* __restrict__ scan, int* __restrict__ index,
                                                      float* __restrict__ alive_opacity, int* __restrict__ n_dead) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int nd = scan[P], d = scan[i];
    if (i == 0) *n_dead = nd;
    const float o = sigmoid(raw_opacity[i]);
    if (o <= min_opacity) {
        index[d] = (int)i;
    } else {
        const int a = (int)i - d;
        index[nd + a] = (int)i;
        alive_opacity[a] = o;
    }
}

// ---- relocate / add: draw counts per source, with the range check of every index
__global__ void __launch_bounds__(256) count_kernel(int P, int n, const int* __restrict__ dead,
                                                    const int* __restrict__ src, int* __restrict__ counts,
                                                    int* __restrict__ err) {
    const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int s = src[j], d = dead ? dead[j] : 0;
    if (s < 0 || s >= P || d < 0 || d >= P) {
        *err = 1;
        return;
    }
    atomicAdd(counts + s, 1);
}

// (raw opacity, raw scaling x3) of every draw's source, from the values before any write (counts not yet scanned)
__global__ void __launch_bounds__(256) relocate_values_kernel(int n, const int* __restrict__ src,
                                                              const float* __restrict__ raw_opacity,
                                                              const float* __restrict__ raw_scaling,
                                                              const int* __restrict__ counts, const int* __restrict__ err,
                                                              float min_opacity, float4* __restrict__ out) {
    const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (j >= n || *err) return;
    const int s = src[j];
    double op, ratio;
    relocation(sigmoid(raw_opacity[s]), copies(counts[s]), op, ratio);
    const float* rs = raw_scaling + 3 * (size_t)s;
    out[j] = make_float4(raw_opacity_of(op, min_opacity), raw_scaling_of(rs[0], ratio), raw_scaling_of(rs[1], ratio),
                         raw_scaling_of(rs[2], ratio));
}

constexpr int kThreads = 256, kPerThread = 8, kChunk = kThreads * kPerThread;

// Segments of a flat pass: one per field (relocate: 7) or per (group, field) (add: 21), each a run of kChunk-element
// blocks over rows of `width` floats
template <int S>
struct Segments {
    int width[S];
    unsigned long long block_end[S];  // exclusive prefix of the segments' block counts
    unsigned long long set(const int w7[7], long long rows) {
        unsigned long long blocks = 0;
        for (int k = 0; k < S; k++) {
            width[k] = w7[k % 7];
            blocks += ((unsigned long long)rows * width[k] + kChunk - 1) / kChunk;
            block_end[k] = blocks;
        }
        return blocks;
    }
    __device__ __forceinline__ int find(unsigned long long& first) const {
        int seg = 0;
        while (blockIdx.x >= block_end[seg]) seg++;
        first = seg ? block_end[seg - 1] : 0ull;
        return seg;
    }
};

struct RelocateArgs {
    Segments<7> seg;
    float *raw[7], *m[7], *v[7];
    const int *dead, *src, *err;
    const float4* values;
    __half* f16;
};

__global__ void __launch_bounds__(kThreads) relocate_apply_kernel(const __grid_constant__ RelocateArgs a, int n) {
    if (*a.err) return;
    unsigned long long first;
    const int field = a.seg.find(first);
    const int w = a.seg.width[field];
    float* __restrict__ raw = a.raw[field];
    float* __restrict__ m = a.m[field];
    float* __restrict__ v = a.v[field];
    const size_t total = (size_t)n * w;
    size_t e = (size_t)(blockIdx.x - first) * kChunk + threadIdx.x;
    size_t j = e / w;
    int col = (int)(e - j * w);
    const int dq = kThreads / w, dr = kThreads % w;
    for (int k = 0; k < kPerThread && e < total; k++, e += kThreads) {
        const size_t s = (size_t)a.src[j] * w + col, d = (size_t)a.dead[j] * w + col;
        float val;
        if (field == kFieldOpacity || field == kFieldScaling) {
            const float4 nv = a.values[j];
            val = field == kFieldOpacity ? nv.x : col == 0 ? nv.y : col == 1 ? nv.z : nv.w;
            raw[s] = val;
        } else {
            val = raw[s];
        }
        raw[d] = val;
        m[s] = 0.0f;
        v[s] = 0.0f;
        if (field == kFieldFeature && a.f16) a.f16[d] = __float2half_rn(val);
        col += dr;
        j += dq;
        if (col >= w) {
            col -= w;
            j++;
        }
    }
}

// ---- add
__global__ void __launch_bounds__(256) fill_lists_kernel(int n, const int* __restrict__ src,
                                                         const int* __restrict__ offsets, int* __restrict__ cursor,
                                                         int* __restrict__ list, const int* __restrict__ err) {
    const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (j >= n || *err) return;
    const int s = src[j];
    list[offsets[s] + atomicAdd(cursor + s, 1)] = (int)j;
}

struct AddArgs {
    Segments<21> seg;
    const float* src[21];
    float* dst[21];
    const int *offsets, *list, *err;
    const float4* values;
};

__global__ void __launch_bounds__(kThreads) add_apply_kernel(const __grid_constant__ AddArgs a, int P) {
    if (*a.err) return;
    unsigned long long first;
    const int sg = a.seg.find(first);
    const int w = a.seg.width[sg], group = sg / 7, field = sg % 7;
    const float* __restrict__ src = a.src[sg];
    float* __restrict__ dst = a.dst[sg];
    const size_t total = (size_t)P * w;
    size_t e = (size_t)(blockIdx.x - first) * kChunk + threadIdx.x;
    size_t row = e / w;
    int col = (int)(e - row * w);
    const int dq = kThreads / w, dr = kThreads % w;
    for (int k = 0; k < kPerThread && e < total; k++, e += kThreads) {
        const int o0 = a.offsets[row], o1 = a.offsets[row + 1];
        float val, copy;
        if (group) {  // moments: zero for drawn rows and new rows
            val = o1 > o0 ? 0.0f : src[e];
            copy = 0.0f;
        } else if (o1 > o0 && (field == kFieldOpacity || field == kFieldScaling)) {
            const float4 nv = a.values[a.list[o0]];  // the values of the row's first draw (all its draws have them)
            val = copy = field == kFieldOpacity ? nv.x : col == 0 ? nv.y : col == 1 ? nv.z : nv.w;
        } else {
            val = copy = src[e];
        }
        dst[e] = val;
        for (int t = o0; t < o1; t++) dst[((size_t)P + a.list[t]) * w + col] = copy;
        col += dr;
        row += dq;
        if (col >= w) {
            col -= w;
            row++;
        }
    }
}

// ---- noise
__global__ void __launch_bounds__(256) noise_kernel(int P, float* __restrict__ xyz, const float* __restrict__ raw_opacity,
                                                    const float* __restrict__ raw_scaling,
                                                    const float* __restrict__ raw_rotation,
                                                    const float* __restrict__ eps, float scale) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= P) return;
    const double o = sigmoid(raw_opacity[i]);
    const double g = 1.0 / (1.0 + exp(-100.0 * ((1.0 - o) - 0.995)));
    const float4 r = reinterpret_cast<const float4*>(raw_rotation)[i];
    const double rw = r.x, rx = r.y, ry = r.z, rz = r.w;
    const double nrm = sqrt(rw * rw + rx * rx + ry * ry + rz * rz);
    const double w = rw / nrm, x = rx / nrm, y = ry / nrm, z = rz / nrm;
    const double R[3][3] = {{1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)},
                            {2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)},
                            {2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)}};
    const double k = g * (double)scale;
    double v[3], t[3];
    for (int c = 0; c < 3; c++) v[c] = (double)eps[3 * i + c] * k;
    for (int c = 0; c < 3; c++) {  // t = diag(s^2) R^T v
        const double s = expf(raw_scaling[3 * i + c]);
        t[c] = s * s * (R[0][c] * v[0] + R[1][c] * v[1] + R[2][c] * v[2]);
    }
    for (int c = 0; c < 3; c++)
        xyz[3 * i + c] = (float)((double)xyz[3 * i + c] + (R[c][0] * t[0] + R[c][1] * t[1] + R[c][2] * t[2]));
}

}  // namespace

cudaError_t mcmc_scratch_bytes(int P, size_t* bytes) {
    *bytes = 0;
    if (P <= 0) return cudaSuccess;
    size_t sb = 0;
    const cudaError_t e = scan_bytes(P, &sb);
    if (e != cudaSuccess) return e;
    *bytes = mcmc_scratch_fixed_bytes(P) + align_up(sb);
    return cudaSuccess;
}

size_t mcmc_scratch_fixed_bytes(int P) {
    return P > 0 ? 256 + align_up(((size_t)P + 1) * 4) + align_up((size_t)P * 24) : 0;
}

cudaError_t launch_mcmc_plan(int P, const float* raw_opacity, float min_opacity, char* scratch, int32_t* n_dead,
                             int32_t* index, float* alive_opacity, cudaStream_t s) {
    if (P == 0) return cudaMemsetAsync(n_dead, 0, sizeof(int32_t), s);
    size_t sb = 0;
    cudaError_t e = scan_bytes(P, &sb);
    if (e != cudaSuccess) return e;
    const Scratch sc(P, scratch);
    classify_kernel<<<blocks_for((long long)P + 1), 256, 0, s>>>(P, raw_opacity, min_opacity, sc.counts);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = cub::DeviceScan::ExclusiveSum(sc.cub, sb, sc.counts, sc.counts, P + 1, s)) != cudaSuccess) return e;
    scatter_kernel<<<blocks_for(P), 256, 0, s>>>(P, raw_opacity, min_opacity, sc.counts, index, alive_opacity, n_dead);
    g_launches++;
    return cudaGetLastError();
}

namespace {
// zero the error flag and the counts, then count (and range-check) the draws
cudaError_t count_draws(int P, int n, const int32_t* dead, const int32_t* src, const Scratch& sc, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(sc.err, 0, 256 + ((size_t)P + 1) * 4, s);
    if (e != cudaSuccess || n == 0) return e;
    count_kernel<<<blocks_for(n), 256, 0, s>>>(P, n, dead, src, sc.counts, sc.err);
    g_launches++;
    return cudaGetLastError();
}
}  // namespace

cudaError_t launch_mcmc_relocate(int P, int M, int C, int n, const int32_t* dead, const int32_t* src, float min_opacity,
                                 float* const fields[21], __half* feature_f16, char* scratch, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const Scratch sc(P, scratch);
    cudaError_t e = count_draws(P, n, dead, src, sc, s);
    if (e != cudaSuccess) return e;
    relocate_values_kernel<<<blocks_for(n), 256, 0, s>>>(n, src, fields[kFieldOpacity], fields[kFieldScaling], sc.counts,
                                                         sc.err, min_opacity, sc.per_draw);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const int width[7] = {3, 3, 3 * (M - 1), 1, 3, 4, C};
    RelocateArgs a;
    const unsigned long long blocks = a.seg.set(width, n);
    for (int k = 0; k < 7; k++) {
        a.raw[k] = fields[k];
        a.m[k] = fields[7 + k];
        a.v[k] = fields[14 + k];
    }
    a.dead = dead; a.src = src; a.err = sc.err; a.values = sc.per_draw; a.f16 = C > 0 ? feature_f16 : nullptr;
    if (blocks > 0x7fffffffull) return cudaErrorInvalidConfiguration;
    relocate_apply_kernel<<<(unsigned)blocks, kThreads, 0, s>>>(a, n);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_mcmc_add(int P, int M, int C, int n, const int32_t* src, float min_opacity,
                            const float* const src_fields[21], float* const dst_fields[21], char* scratch,
                            cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    size_t sb = 0;
    cudaError_t e = scan_bytes(P, &sb);
    if (e != cudaSuccess) return e;
    const Scratch sc(P, scratch);
    if ((e = count_draws(P, n, nullptr, src, sc, s)) != cudaSuccess) return e;
    if (n > 0) {
        relocate_values_kernel<<<blocks_for(n), 256, 0, s>>>(n, src, src_fields[kFieldOpacity],
                                                             src_fields[kFieldScaling], sc.counts, sc.err, min_opacity,
                                                             sc.per_draw);
        g_launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    if ((e = cub::DeviceScan::ExclusiveSum(sc.cub, sb, sc.counts, sc.counts, P + 1, s)) != cudaSuccess) return e;
    if (n > 0) {
        if ((e = cudaMemsetAsync(sc.cursor, 0, (size_t)P * 4, s)) != cudaSuccess) return e;
        fill_lists_kernel<<<blocks_for(n), 256, 0, s>>>(n, src, sc.counts, sc.cursor, sc.list, sc.err);
        g_launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    const int width[7] = {3, 3, 3 * (M - 1), 1, 3, 4, C};
    AddArgs a;
    const unsigned long long blocks = a.seg.set(width, P);
    for (int k = 0; k < 21; k++) {
        a.src[k] = src_fields[k];
        a.dst[k] = dst_fields[k];
    }
    a.offsets = sc.counts; a.list = sc.list; a.err = sc.err; a.values = sc.per_draw;
    if (blocks > 0x7fffffffull) return cudaErrorInvalidConfiguration;
    add_apply_kernel<<<(unsigned)blocks, kThreads, 0, s>>>(a, P);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_mcmc_inject_noise(int P, float* xyz, const float* raw_opacity, const float* raw_scaling,
                                     const float* raw_rotation, const float* eps, float scale, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    noise_kernel<<<blocks_for(P), 256, 0, s>>>(P, xyz, raw_opacity, raw_scaling, raw_rotation, eps, scale);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace f3dgs
