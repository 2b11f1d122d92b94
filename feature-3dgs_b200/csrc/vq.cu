// Vector quantisation of per-row features (LightGaussian, CompGS): a codebook c [K, D] and one code per row of
// x [P, D] (include/f3dgs_b200.h: f3dgs_vq_*).
//
//   assign   code[i] = argmin_k (||c_k||^2 - 2 x_i . c_k).  A prep kernel rounds the codebook to TF32 into [Kp, Dp]
//            (zero-padded to whole tiles) and sums ||c_k||^2 in fp32 from the unrounded rows, one warp per code in a
//            fixed order.  The main kernel is a TF32 mma.sync GEMM whose epilogue keeps a running minimum per row: a
//            CTA owns 128 rows, walks the codes in chunks of 128 and D in steps of 32 channels, with the x slice and
//            the codebook slice of a step double-buffered in shared memory by cp.async; its 8 warps are 4 (rows) x 2
//            (codes), each with a 32 x 64 accumulator tile.  x is rounded to TF32 as fragments are read.  Only the codes
//            reach memory.
//   plan     a stable sort of the row indices by code (cub radix sort over the code's bits) and the segment offsets
//            offsets[k] = lower_bound(sorted codes, k), in the caller's scratch.  An out-of-range code raises the
//            plan's error flag; every later update or gradient over that plan then writes nothing.
//   reduce   the rows of each code, summed in double: phase 1 sums each chunk of kChunkRows sorted rows that lies
//            inside one code (one CTA per chunk); phase 2 gives each (code, column tile) its head rows, the sums of its
//            whole chunks, then its tail rows, in that order.  No CTA sums more than 2 kChunkRows rows plus P /
//            kChunkRows chunk sums per column, so one code holding every row is spread over P / kChunkRows CTAs.  No
//            float atomics; the order depends on P and the codes only.
//   decode   out[i] = c[code[i]], float32 or half_rn, one thread per 16-byte store where D allows it.
// Every kernel is bitwise reproducible for equal inputs.
#include <cub/cub.cuh>

#include <cfloat>
#include <cmath>
#include <type_traits>

#include "kernels.h"
#include "tf32_mma.cuh"

namespace f3dgs {

namespace {

// ---------------------------------------------------------------------------------------------------- assign
constexpr int kAWarps = 8, kAThreads = 32 * kAWarps;
constexpr int kBM = 128, kBN = 128, kBK = 32;  // rows per CTA, codes per chunk, channels per step
constexpr int kLd = kBK + 4;                    // shared row stride: conflict-free fragment reads
constexpr int kTileFloats = kBM * kLd;          // one x or codebook slice
constexpr size_t kAssignSmem = 4 * kTileFloats * sizeof(float);  // x and codebook, two stages each

template <int B>  // zero-filling cp.async of B = 4 or 16 bytes
__device__ __forceinline__ void cp_async_zfill(float* dst, const float* src, bool valid) {
    const int n = valid ? B : 0;
    if constexpr (B == 16)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(n) : "memory");
    else
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(n) : "memory");
}

// (vb, ib) replaces (va, ia) as the minimum: a number beats NaN, ties go to the lower index.  A strict preference, so
// the two lanes of a shuffle pair pick the same winner.
__device__ __forceinline__ bool beats_min(float vb, int ib, float va, int ia) {
    if (va != va) return vb == vb || ib < ia;
    return vb < va || (vb == va && ib < ia);
}

// one warp per padded code r: cr[r] = c_r rounded to TF32 (zero past K and D), cn[r] = ||c_r||^2 in fp32 (lane-strided
// partial sums, then a fixed shuffle tree)
__global__ void assign_prep_kernel(int K, int D, int Dp, const float* __restrict__ c, float* __restrict__ cr,
                                   float* __restrict__ cn) {
    const int r = blockIdx.x, lane = threadIdx.x;
    const float* row = c + (size_t)r * D;
    float ss = 0.f;
    if (r < K)
        for (int d = lane; d < D; d += 32) ss = fmaf(row[d], row[d], ss);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    for (int d = lane; d < Dp; d += 32)
        cr[(size_t)r * Dp + d] = __uint_as_float(to_tf32(r < K && d < D ? row[d] : 0.f));
    if (lane == 0) cn[r] = ss;
}

template <int V>  // V = 4: D % 4 == 0 and 16-byte x rows, loaded by 16-byte copies; V = 1: by 4-byte copies
__global__ void __launch_bounds__(kAThreads, 2)
    assign_kernel(int P, int K, int D, int Dp, const float* __restrict__ x, const float* __restrict__ cr,
                  const float* __restrict__ cn, int32_t* __restrict__ code) {
    extern __shared__ float4 smem4[];
    float* xs = reinterpret_cast<float*>(smem4);  // [2][kBM][kLd]
    float* cs = xs + 2 * kTileFloats;             // [2][kBN][kLd]
    __shared__ float red_v[kBM];
    __shared__ int red_i[kBM];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    const long long row0 = (long long)blockIdx.x * kBM;
    const int steps = Dp / kBK, chunks = (K + kBN - 1) / kBN, stages = steps * chunks;

    auto load_stage = [&](int q) {
        const int ch = q / steps, k0 = (q - ch * steps) * kBK;
        float* xd = xs + (q & 1) * kTileFloats;
        for (int i = threadIdx.x; i < kBM * kBK / V; i += kAThreads) {
            const int r = i / (kBK / V), col = k0 + (i - r * (kBK / V)) * V;
            const long long row = row0 + r;
            const bool ok = row < P && col < D;
            cp_async_zfill<4 * V>(xd + r * kLd + col - k0, ok ? x + row * D + col : x, ok);
        }
        const float* src = cr + (size_t)ch * kBN * Dp + k0;
        float* cd = cs + (q & 1) * kTileFloats;
        for (int i = threadIdx.x; i < kBN * kBK / 4; i += kAThreads) {
            const int r = i / (kBK / 4), col = (i - r * (kBK / 4)) * 4;
            cp_async16(cd + r * kLd + col, src + (size_t)r * Dp + col);
        }
        cp_async_commit();
    };
    load_stage(0);

    // running minimum of this lane's rows (mi, half): wm * 32 + 16 mi + g + 8 half
    float best[4];
    int arg[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        best[j] = __int_as_float(0x7fc00000);
        arg[j] = 0x7fffffff;
    }
    float acc[2][8][4];

    for (int q = 0; q < stages; q++) {
        const int ch = q / steps, st = q - ch * steps;
        if (st == 0) {
#pragma unroll
            for (int mi = 0; mi < 2; mi++)
#pragma unroll
                for (int nj = 0; nj < 8; nj++)
#pragma unroll
                    for (int i = 0; i < 4; i++) acc[mi][nj][i] = 0.f;
        }
        cp_async_wait_all();
        __syncthreads();  // stage q has landed, and every warp is done with the buffers stage q + 1 overwrites
        if (q + 1 < stages) load_stage(q + 1);
        const float* xa = xs + (q & 1) * kTileFloats + (wm * 32 + g) * kLd + t;
        const float* cb = cs + (q & 1) * kTileFloats + (wn * 64 + g) * kLd + t;
#pragma unroll
        for (int kk = 0; kk < kBK; kk += 8) {
            uint32_t a[2][4];
#pragma unroll
            for (int mi = 0; mi < 2; mi++) {
                const float* p = xa + mi * 16 * kLd + kk;
                a[mi][0] = to_tf32(p[0]);
                a[mi][1] = to_tf32(p[8 * kLd]);
                a[mi][2] = to_tf32(p[4]);
                a[mi][3] = to_tf32(p[8 * kLd + 4]);
            }
#pragma unroll
            for (int nj = 0; nj < 8; nj++) {
                const float* p = cb + nj * 8 * kLd + kk;
                const uint32_t b0 = __float_as_uint(p[0]), b1 = __float_as_uint(p[4]);
                mma_tf32(acc[0][nj], a[0], b0, b1);
                mma_tf32(acc[1][nj], a[1], b0, b1);
            }
        }
        if (st != steps - 1) continue;

        // chunk epilogue: score = ||c_k||^2 - 2 x . c_k, codes in increasing order per lane
#pragma unroll
        for (int nj = 0; nj < 8; nj++) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int k = ch * kBN + wn * 64 + nj * 8 + 2 * t + h;
                if (k >= K) continue;
                const float n2 = __ldg(cn + k);
#pragma unroll
                for (int mi = 0; mi < 2; mi++)
#pragma unroll
                    for (int hr = 0; hr < 2; hr++) {
                        const float s = n2 - 2.f * acc[mi][nj][2 * hr + h];
                        if (beats_min(s, k, best[2 * mi + hr], arg[2 * mi + hr])) {
                            best[2 * mi + hr] = s;
                            arg[2 * mi + hr] = k;
                        }
                    }
            }
        }
    }

    // the 4 lanes of a quad share rows; then the two code halves of the CTA meet in shared memory
#pragma unroll
    for (int j = 0; j < 4; j++) {
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best[j], o);
            const int oi = __shfl_xor_sync(0xffffffffu, arg[j], o);
            if (beats_min(ob, oi, best[j], arg[j])) {
                best[j] = ob;
                arg[j] = oi;
            }
        }
    }
    if (wn == 1 && t == 0) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int r = wm * 32 + 16 * (j >> 1) + g + 8 * (j & 1);
            red_v[r] = best[j];
            red_i[r] = arg[j];
        }
    }
    __syncthreads();
    if (wn == 0 && t == 0) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int r = wm * 32 + 16 * (j >> 1) + g + 8 * (j & 1);
            if (beats_min(red_v[r], red_i[r], best[j], arg[j])) arg[j] = red_i[r];
            if (row0 + r < P) code[row0 + r] = arg[j];
        }
    }
}

// ---------------------------------------------------------------------------------------------------- plan
constexpr int kChunkRows = 256;  // sorted rows per phase-1 chunk

// scratch: [flags 256 B | sorted codes uint32 [P] | order int32 [P] | offsets int32 [K + 1] | iota int32 [P] | cub]
struct Plan {
    int* err;
    uint32_t* sorted;
    int *order, *offsets, *iota;
    char* cub;
    Plan(int P, int K, char* base) {
        err = reinterpret_cast<int*>(base);
        size_t o = 256;
        sorted = reinterpret_cast<uint32_t*>(base + o);  o += align_up((size_t)P * 4);
        order = reinterpret_cast<int*>(base + o);        o += align_up((size_t)P * 4);
        offsets = reinterpret_cast<int*>(base + o);      o += align_up(((size_t)K + 1) * 4);
        iota = reinterpret_cast<int*>(base + o);         o += align_up((size_t)P * 4);
        cub = base + o;
    }
    static size_t fixed_bytes(int P, int K) {
        return 256 + 3 * align_up((size_t)P * 4) + align_up(((size_t)K + 1) * 4);
    }
};

int code_bits(int K) {
    int b = 1;
    while (b < 31 && (1u << b) < (unsigned)K) b++;
    return b;
}

cudaError_t sort_bytes(int P, int K, size_t* bytes) {
    *bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                           (const int*)nullptr, (int*)nullptr, P, 0, code_bits(K));
}

__global__ void __launch_bounds__(256) plan_check_kernel(int P, int K, const int32_t* __restrict__ code,
                                                         int* __restrict__ iota, int* __restrict__ err) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= P) return;
    iota[i] = (int)i;
    const int c = code[i];
    if (c < 0 || c >= K) atomicOr(err, 1);
}

__global__ void __launch_bounds__(256) plan_offsets_kernel(int P, int K, const uint32_t* __restrict__ sorted,
                                                           int* __restrict__ offsets) {
    const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (k > K) return;
    int lo = 0, hi = P;  // first position whose code is >= k
    while (lo < hi) {
        const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
        if (sorted[mid] < (uint32_t)k) lo = mid + 1;
        else hi = mid;
    }
    offsets[k] = lo;
}

// ---------------------------------------------------------------------------------------------------- reduce
// per-call flags and partials: [flags 256 B | chunk weight sums double [T] | chunk sums double [T, D]]
constexpr int kRedThreads = 128;  // phase 2: columns per CTA

__global__ void __launch_bounds__(256) weight_check_kernel(int P, const float* __restrict__ w, int* __restrict__ err) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float v = w[i];
    if (!(v >= 0.f && v <= FLT_MAX)) atomicOr(err, 1);  // NaN, negative or infinite
}

// phase 1: the sums of the chunks that lie inside one code
__global__ void __launch_bounds__(256) chunk_sum_kernel(int P, int D, const float* __restrict__ x,
                                                        const float* __restrict__ w, const uint32_t* __restrict__ sorted,
                                                        const int* __restrict__ order, const int* __restrict__ plan_err,
                                                        const int* __restrict__ werr, double* __restrict__ part_w,
                                                        double* __restrict__ part) {
    __shared__ int rows[kChunkRows];
    __shared__ float ws[kChunkRows];
    if (*plan_err || *werr) return;
    const int c = blockIdx.x, r0 = c * kChunkRows, n = min(kChunkRows, P - r0);
    if (sorted[r0] != sorted[r0 + n - 1]) return;
    for (int r = threadIdx.x; r < n; r += blockDim.x) {
        rows[r] = order[r0 + r];
        ws[r] = w ? w[rows[r]] : 1.f;
    }
    __syncthreads();
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        double s = 0.0;
        for (int r = 0; r < n; r++) s += (double)ws[r] * (double)x[(size_t)rows[r] * D + d];
        part[(size_t)c * D + d] = s;
    }
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int r = 0; r < n; r++) s += (double)ws[r];
        part_w[c] = s;
    }
}

// phase 2: one CTA per (code, tile of kRedThreads columns).  MEAN: out[k] = sum w x / sum w where sum w > 0 (else the
// row is left as it is); otherwise out[k] = sum x, written for every code
template <bool MEAN>
__global__ void __launch_bounds__(kRedThreads) segment_kernel(int D, const float* __restrict__ x,
                                                              const float* __restrict__ w, const int* __restrict__ order,
                                                              const int* __restrict__ offsets,
                                                              const int* __restrict__ plan_err,
                                                              const int* __restrict__ werr,
                                                              const double* __restrict__ part_w,
                                                              const double* __restrict__ part, float* __restrict__ out) {
    if (*plan_err || *werr) return;
    const int k = blockIdx.x, d = blockIdx.y * kRedThreads + threadIdx.x;
    if (d >= D) return;
    const int o = offsets[k], e = offsets[k + 1];
    const int cf = (o + kChunkRows - 1) / kChunkRows, cl = e / kChunkRows;  // whole chunks [cf, cl)
    const bool whole = cf < cl;
    const int head_end = whole ? cf * kChunkRows : e, tail_begin = whole ? cl * kChunkRows : e;
    double s = 0.0, sw = 0.0;
    auto rows = [&](int a, int b) {
        for (int r = a; r < b; r++) {
            const int i = __ldg(order + r);
            const double wi = w ? (double)__ldg(w + i) : 1.0;
            s += wi * (double)__ldg(x + (size_t)i * D + d);
            sw += wi;
        }
    };
    rows(o, head_end);
    for (int c = cf; c < cl; c++) {
        s += part[(size_t)c * D + d];
        sw += part_w[c];
    }
    rows(tail_begin, e);
    if (MEAN) {
        if (sw > 0.0) out[(size_t)k * D + d] = (float)(s / sw);
    } else {
        out[(size_t)k * D + d] = (float)s;
    }
}

// ---------------------------------------------------------------------------------------------------- decode
// V elements per thread (V = 8 for float16 and 4 for float32 when D is a multiple of V, else 1).  A code outside
// [0, K) decodes to a NaN row.
template <typename T, int V>
__global__ void __launch_bounds__(256) decode_kernel(long long n, int K, int D, const float* __restrict__ c,
                                                     const int32_t* __restrict__ code, T* __restrict__ out) {
    const long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x;  // vector index
    if (v >= n) return;
    const long long e = v * V;
    const long long i = e / D;
    const int col = (int)(e - i * D);
    const int k = __ldg(code + i);
    const bool ok = k >= 0 && k < K;
    float f[V];
    const float* src = c + (size_t)(ok ? k : 0) * D + col;
    if constexpr (V >= 4) {
#pragma unroll
        for (int j = 0; j < V; j += 4) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(src + j));
            f[j] = q.x; f[j + 1] = q.y; f[j + 2] = q.z; f[j + 3] = q.w;
        }
    } else {
        f[0] = __ldg(src);
    }
    if (!ok)
#pragma unroll
        for (int j = 0; j < V; j++) f[j] = __int_as_float(0x7fc00000);
    if constexpr (std::is_same<T, float>::value) {
        if constexpr (V == 4) reinterpret_cast<float4*>(out)[v] = make_float4(f[0], f[1], f[2], f[3]);
        else out[e] = f[0];
    } else {
        if constexpr (V == 8) {
            uint4 u;
            __half2 h[4];
#pragma unroll
            for (int j = 0; j < 4; j++) h[j] = __halves2half2(__float2half_rn(f[2 * j]), __float2half_rn(f[2 * j + 1]));
            u = *reinterpret_cast<const uint4*>(h);
            reinterpret_cast<uint4*>(out)[v] = u;
        } else {
            out[e] = __float2half_rn(f[0]);
        }
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------- launchers
cudaError_t launch_vq_assign(int P, int K, int D, const float* x, const float* codebook, int32_t* code,
                             cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    const int Kp = (int)align_up((size_t)K, kBN), Dp = (int)align_up((size_t)D, kBK);
    const size_t off_n = align_up((size_t)Kp * Dp * 4, 256);
    char* ws = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&ws, off_n + (size_t)Kp * 4, s);
    if (e != cudaSuccess) return e;
    float* cr = reinterpret_cast<float*>(ws);
    float* cn = reinterpret_cast<float*>(ws + off_n);
    assign_prep_kernel<<<Kp, 32, 0, s>>>(K, D, Dp, codebook, cr, cn);
    g_launches++;
    e = cudaGetLastError();
    if (e == cudaSuccess) {
        const bool vec = D % 4 == 0 && ((uintptr_t)x & 15) == 0;
        auto kernel = vec ? assign_kernel<4> : assign_kernel<1>;
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAssignSmem);
        if (e == cudaSuccess) {
            const unsigned grid = (unsigned)(((size_t)P + kBM - 1) / kBM);
            kernel<<<grid, kAThreads, kAssignSmem, s>>>(P, K, D, Dp, x, cr, cn, code);
            g_launches++;
            e = cudaGetLastError();
        }
    }
    cudaFreeAsync(ws, s);
    return e;
}

size_t vq_scratch_fixed_bytes(int P, int K) { return P > 0 ? Plan::fixed_bytes(P, K) : 0; }

cudaError_t vq_scratch_bytes(int P, int K, size_t* bytes) {
    *bytes = 0;
    if (P <= 0) return cudaSuccess;
    size_t sb = 0;
    const cudaError_t e = sort_bytes(P, K, &sb);
    if (e != cudaSuccess) return e;
    *bytes = Plan::fixed_bytes(P, K) + align_up(sb);
    return cudaSuccess;
}

cudaError_t launch_vq_plan(int P, int K, const int32_t* code, char* scratch, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    size_t sb = 0;
    cudaError_t e = sort_bytes(P, K, &sb);
    if (e != cudaSuccess) return e;
    const Plan pl(P, K, scratch);
    if ((e = cudaMemsetAsync(pl.err, 0, 4, s)) != cudaSuccess) return e;
    plan_check_kernel<<<blocks_for(P), 256, 0, s>>>(P, K, code, pl.iota, pl.err);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    e = cub::DeviceRadixSort::SortPairs(pl.cub, sb, reinterpret_cast<const uint32_t*>(code), pl.sorted, pl.iota,
                                        pl.order, P, 0, code_bits(K), s);
    if (e != cudaSuccess) return e;
    plan_offsets_kernel<<<blocks_for((long long)K + 1), 256, 0, s>>>(P, K, pl.sorted, pl.offsets);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_vq_reduce(int P, int K, int D, const float* x, const float* weights, const char* scratch, float* out,
                             bool mean, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    const Plan pl(P, K, const_cast<char*>(scratch));
    const int T = (P + kChunkRows - 1) / kChunkRows;
    const size_t off_part = 256 + align_up((size_t)T * 8);
    char* ws = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&ws, off_part + (size_t)T * D * 8, s);
    if (e != cudaSuccess) return e;
    int* werr = reinterpret_cast<int*>(ws);
    double* part_w = reinterpret_cast<double*>(ws + 256);
    double* part = reinterpret_cast<double*>(ws + off_part);
    e = cudaMemsetAsync(werr, 0, 4, s);
    if (e == cudaSuccess && weights) {
        weight_check_kernel<<<blocks_for(P), 256, 0, s>>>(P, weights, werr);
        g_launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        chunk_sum_kernel<<<T, 256, 0, s>>>(P, D, x, weights, pl.sorted, pl.order, pl.err, werr, part_w, part);
        g_launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        const dim3 grid((unsigned)K, (unsigned)((D + kRedThreads - 1) / kRedThreads));
        if (mean)
            segment_kernel<true><<<grid, kRedThreads, 0, s>>>(D, x, weights, pl.order, pl.offsets, pl.err, werr, part_w,
                                                              part, out);
        else
            segment_kernel<false><<<grid, kRedThreads, 0, s>>>(D, x, nullptr, pl.order, pl.offsets, pl.err, werr,
                                                               part_w, part, out);
        g_launches++;
        e = cudaGetLastError();
    }
    cudaFreeAsync(ws, s);
    return e;
}

template <typename T>
cudaError_t launch_vq_decode(int P, int K, int D, const float* codebook, const int32_t* code, T* out, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    constexpr int VW = std::is_same<T, float>::value ? 4 : 8;
    const long long total = (long long)P * D;
    const bool vec = D % VW == 0 && ((uintptr_t)codebook & 15) == 0 && ((uintptr_t)out & 15) == 0;
    const long long n = vec ? total / VW : total;
    const long long blocks = (n + 255) / 256;
    if (blocks > 0x7fffffffll) return cudaErrorInvalidConfiguration;
    if (vec)
        decode_kernel<T, VW><<<(unsigned)blocks, 256, 0, s>>>(n, K, D, codebook, code, out);
    else
        decode_kernel<T, 1><<<(unsigned)blocks, 256, 0, s>>>(n, K, D, codebook, code, out);
    g_launches++;
    return cudaGetLastError();
}
template cudaError_t launch_vq_decode(int, int, int, const float*, const int32_t*, float*, cudaStream_t);
template cudaError_t launch_vq_decode(int, int, int, const float*, const int32_t*, __half*, cudaStream_t);

}  // namespace f3dgs
