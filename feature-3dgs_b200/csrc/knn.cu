// Exact 3-nearest-neighbour mean squared distance: the initial Gaussian scale of create_from_pcd
// (reference scene/gaussian_model.py:133-160, submodules/simple-knn distCUDA2).
//
//   out[i] = (d0 + d1 + d2) / 3   with d0 <= d1 <= d2 the three smallest squared distances from point i to the points
//                                 j != i (exclusion by index: coincident points count as 0); FLT_MAX fills the
//                                 missing ones when P < 4, as in the reference.
//
// Pipeline (stream-ordered, no host sync; every size below is a function of P alone):
//   1. bbox_kernel     bounding box of the cloud (order-preserving float -> uint encoding, atomicMin/Max: exact and
//                      order-independent)
//   2. morton_kernel   63-bit Morton key (21 bits per axis over the box) and the identity index
//   3. cub::DeviceRadixSort of (key, index) over bits [0, 63)
//   4. leaf_kernel     gathers the points into sorted order (float4) and reduces the AABB of every leaf of 32 points
//   5. node_kernel     one launch per level of the implicit 32-ary hierarchy: node n of level l owns children
//                      [32n, 32n + 32) of level l - 1; its AABB is the union of theirs
//   6. query_kernel    one warp per leaf (32 queries that are close in Morton order): the best-3 of every lane are
//                      seeded from its own leaf, then the warp walks the hierarchy depth-first without a stack and
//                      enters a node only if some lane's AABB distance is below its current third-best distance.
//
// Exactness: a box is pruned only if its distance is not below d2.  The box distance uses the same rounded
// expression as a point distance, and rounding is monotone, so it is a lower bound on the computed distance of every
// point inside; a pruned box cannot change the three smallest values.  Results are bitwise reproducible and independent
// of the input order: every pair distance is one fixed expression of (query, candidate), the best-3 multiset of values
// does not depend on visiting order, and the sum is (d0 + d1) + d2 in ascending order.  No float atomics touch the
// result.
#include <cub/cub.cuh>

#include <algorithm>
#include <cfloat>

#include "kernels.h"

namespace f3dgs {

namespace {

constexpr int kLeaf = 32;       // points per leaf and children per node: one warp lane each
constexpr int kMaxLevels = 8;   // P < 2^31 -> at most 2^26 leaves -> 7 levels above the points

struct KnnLevels {
    int n;                      // number of levels (level 0 = leaves, level n - 1 = the single root)
    int count[kMaxLevels];      // nodes per level
    long long off[kMaxLevels];  // first node of each level in the box arrays
};

KnnLevels knn_levels(int P) {
    KnnLevels L{};
    int c = (P + kLeaf - 1) / kLeaf;
    long long o = 0;
    while (true) {
        L.count[L.n] = c;
        L.off[L.n] = o;
        o += c;
        L.n++;
        if (c <= 1) break;
        c = (c + kLeaf - 1) / kLeaf;
    }
    return L;
}

struct KnnLayout {
    KnnLevels lv;
    size_t bbox, keys_in, keys_out, idx_in, idx_out, pts, box_lo, box_hi, sort_tmp, fixed_bytes;
    explicit KnnLayout(int P) : lv(knn_levels(P)) {
        const size_t n = (size_t)P;
        const size_t nodes = (size_t)(lv.off[lv.n - 1] + lv.count[lv.n - 1]);
        size_t o = 0;
        bbox = o;      o = align_up(o + 6 * sizeof(uint32_t));
        keys_in = o;   o = align_up(o + n * sizeof(uint64_t));
        keys_out = o;  o = align_up(o + n * sizeof(uint64_t));
        idx_in = o;    o = align_up(o + n * sizeof(uint32_t));
        idx_out = o;   o = align_up(o + n * sizeof(uint32_t));
        pts = o;       o = align_up(o + n * sizeof(float4));
        box_lo = o;    o = align_up(o + nodes * sizeof(float4));
        box_hi = o;    o = align_up(o + nodes * sizeof(float4));
        sort_tmp = o;  // CUB's temporary storage goes last: its size needs a device query
        fixed_bytes = o;
    }
};

cudaError_t sort_bytes(int P, size_t* bytes) {
    *bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                           (const uint32_t*)nullptr, (uint32_t*)nullptr, P, 0, 63);
}

// order-preserving map of finite floats onto uint32 (NaN never reaches it)
__device__ __forceinline__ uint32_t ordered(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unordered(uint32_t u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// squared distance of one (query, candidate) pair; the only expression used for it, and for box distances
__device__ __forceinline__ float sq3(float dx, float dy, float dz) {
    return __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
}

__device__ __forceinline__ void insert3(float d, float& d0, float& d1, float& d2) {
    if (d < d2) {
        if (d < d1) {
            d2 = d1;
            if (d < d0) {
                d1 = d0;
                d0 = d;
            } else {
                d1 = d;
            }
        } else {
            d2 = d;
        }
    }
}

__global__ void __launch_bounds__(256) bbox_kernel(int P, const float* __restrict__ pts, uint32_t* __restrict__ bbox) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x)
        for (int a = 0; a < 3; a++) {
            const float v = pts[3 * i + a];
            if (v >= -FLT_MAX && v <= FLT_MAX) {  // finite only: a NaN or inf coordinate does not stretch the box
                lo[a] = fminf(lo[a], v);
                hi[a] = fmaxf(hi[a], v);
            }
        }
    for (int a = 0; a < 3; a++)
        for (int s = 16; s > 0; s >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], s));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], s));
        }
    if ((threadIdx.x & 31) == 0)
        for (int a = 0; a < 3; a++) {
            atomicMin(bbox + a, ordered(lo[a]));
            atomicMax(bbox + 3 + a, ordered(hi[a]));
        }
}

__device__ __forceinline__ uint64_t spread21(uint32_t v) {  // bit k -> bit 3k
    uint64_t x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

__global__ void __launch_bounds__(256) morton_kernel(int P, const float* __restrict__ pts,
                                                     const uint32_t* __restrict__ bbox, uint64_t* __restrict__ keys,
                                                     uint32_t* __restrict__ idx) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= P) return;
    uint64_t key = 0;
    for (int a = 0; a < 3; a++) {
        const float lo = unordered(bbox[a]), hi = unordered(bbox[3 + a]);
        const float ext = hi - lo;
        // zero extent (all points share this coordinate) or overflow: the axis contributes nothing to the order
        const float scale = (ext > 0.f && ext <= FLT_MAX) ? 2097151.f / ext : 0.f;
        const float q = fminf(fmaxf((pts[3 * i + a] - lo) * scale, 0.f), 2097151.f);  // NaN -> 0
        key |= spread21((uint32_t)q) << a;
    }
    keys[i] = key;
    idx[i] = (uint32_t)i;
}

// one warp per leaf: gather its 32 points into sorted order and write the leaf's AABB
__global__ void __launch_bounds__(256) leaf_kernel(int P, const float* __restrict__ pts,
                                                   const uint32_t* __restrict__ order, float4* __restrict__ sorted,
                                                   float4* __restrict__ box_lo, float4* __restrict__ box_hi) {
    const int lane = threadIdx.x & 31;
    const long long leaf = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    const long long i = leaf * kLeaf + lane;
    if (leaf * kLeaf >= P) return;
    float3 lo = make_float3(FLT_MAX, FLT_MAX, FLT_MAX), hi = make_float3(-FLT_MAX, -FLT_MAX, -FLT_MAX);
    if (i < P) {
        const uint32_t j = order[i];
        const float x = pts[3 * (size_t)j], y = pts[3 * (size_t)j + 1], z = pts[3 * (size_t)j + 2];
        sorted[i] = make_float4(x, y, z, 0.f);
        lo = make_float3(x, y, z);
        hi = lo;
    }
    for (int s = 16; s > 0; s >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, s));
        lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, s));
        lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, s));
        hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, s));
        hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, s));
        hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, s));
    }
    if (lane == 0) {
        box_lo[leaf] = make_float4(lo.x, lo.y, lo.z, 0.f);
        box_hi[leaf] = make_float4(hi.x, hi.y, hi.z, 0.f);
    }
}

// one warp per node of a level: the union of its (up to) 32 children's AABBs
__global__ void __launch_bounds__(256) node_kernel(int n_children, const float4* __restrict__ child_lo,
                                                   const float4* __restrict__ child_hi, float4* __restrict__ lo_out,
                                                   float4* __restrict__ hi_out) {
    const int lane = threadIdx.x & 31;
    const long long node = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    const long long c = node * kLeaf + lane;
    if (node * kLeaf >= n_children) return;
    float4 lo = make_float4(FLT_MAX, FLT_MAX, FLT_MAX, 0.f), hi = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, 0.f);
    if (c < n_children) {
        lo = child_lo[c];
        hi = child_hi[c];
    }
    for (int s = 16; s > 0; s >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, s));
        lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, s));
        lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, s));
        hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, s));
        hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, s));
        hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, s));
    }
    if (lane == 0) {
        lo_out[node] = lo;
        hi_out[node] = hi;
    }
}

// best-3 update of every lane against the points of one leaf (all lanes take part; `self` is the lane's sorted index)
__device__ __forceinline__ void scan_leaf(int P, long long leaf, const float4* __restrict__ sorted, int lane,
                                          long long self, float3 q, bool active, float& d0, float& d1, float& d2) {
    const long long base = leaf * kLeaf;
    const int cnt = (int)min((long long)kLeaf, (long long)P - base);
    float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane < cnt) c = sorted[base + lane];
    for (int j = 0; j < cnt; j++) {
        const float cx = __shfl_sync(0xffffffffu, c.x, j);
        const float cy = __shfl_sync(0xffffffffu, c.y, j);
        const float cz = __shfl_sync(0xffffffffu, c.z, j);
        if (active && base + j != self) insert3(sq3(__fsub_rn(cx, q.x), __fsub_rn(cy, q.y), __fsub_rn(cz, q.z)), d0, d1, d2);
    }
}

// distance from q to the box [lo, hi] (0 inside), with the rounding of sq3 on per-axis gaps that are rounded like
// the point differences they bound
__device__ __forceinline__ float box_dist(float3 q, float4 lo, float4 hi) {
    const float gx = q.x < lo.x ? __fsub_rn(lo.x, q.x) : (q.x > hi.x ? __fsub_rn(q.x, hi.x) : 0.f);
    const float gy = q.y < lo.y ? __fsub_rn(lo.y, q.y) : (q.y > hi.y ? __fsub_rn(q.y, hi.y) : 0.f);
    const float gz = q.z < lo.z ? __fsub_rn(lo.z, q.z) : (q.z > hi.z ? __fsub_rn(q.z, hi.z) : 0.f);
    return sq3(gx, gy, gz);
}

// nodes on level l: ceil(P / 32^(l+1)) (nested ceilings of a division by 32 collapse into one)
__device__ __forceinline__ long long level_count(int P, int l) {
    const int sh = 5 * (l + 1);
    return ((long long)P + (1ll << sh) - 1) >> sh;
}

__global__ void __launch_bounds__(256) query_kernel(int P, int top, long long top_off, const float4* __restrict__ sorted,
                                                    const uint32_t* __restrict__ order, const float4* __restrict__ box_lo,
                                                    const float4* __restrict__ box_hi, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long leaf = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    if (leaf * kLeaf >= P) return;  // warp-uniform
    const long long self = leaf * kLeaf + lane;
    const bool active = self < P;
    float3 q = make_float3(0.f, 0.f, 0.f);
    if (active) {
        const float4 p = sorted[self];
        q = make_float3(p.x, p.y, p.z);
    }
    float d0 = FLT_MAX, d1 = FLT_MAX, d2 = FLT_MAX;
    scan_leaf(P, leaf, sorted, lane, self, q, active, d0, d1, d2);

    // stackless depth-first walk from the root: (l, n) is the current node, its siblings are n + 1 while n % 32 != 31;
    // level l's boxes start at `off`, and level l - 1's right before them (levels are stored leaves first)
    int l = top;
    long long n = 0, off = top_off, cnt = 1;
    while (true) {
        const bool need = active && box_dist(q, box_lo[off + n], box_hi[off + n]) < d2;
        if (__any_sync(0xffffffffu, need)) {
            if (l > 0) {  // enter: first child
                l--;
                n *= kLeaf;
                cnt = level_count(P, l);
                off -= cnt;
                continue;
            }
            if (n != leaf) scan_leaf(P, n, sorted, lane, self, q, active, d0, d1, d2);
        }
        // next node in depth-first order: the next sibling, else the parent's next sibling, ...
        while (l < top && ((n & (kLeaf - 1)) == kLeaf - 1 || n + 1 >= cnt)) {
            off += cnt;
            l++;
            n >>= 5;
            cnt = level_count(P, l);
        }
        if (l == top) break;
        n++;
    }
    if (active) out[order[self]] = __fdiv_rn(__fadd_rn(__fadd_rn(d0, d1), d2), 3.f);
}

}  // namespace

cudaError_t knn_scratch_bytes(int P, size_t* bytes) {
    *bytes = 0;
    if (P <= 0) return cudaSuccess;
    size_t sb = 0;
    const cudaError_t e = sort_bytes(P, &sb);
    if (e != cudaSuccess) return e;
    *bytes = KnnLayout(P).fixed_bytes + align_up(sb);
    return cudaSuccess;
}

size_t knn_scratch_fixed_bytes(int P) { return P > 0 ? KnnLayout(P).fixed_bytes : 0; }

cudaError_t launch_knn_mean_dist(int P, const float* points, float* out, char* scratch, cudaStream_t s) {
    if (P <= 0) return cudaSuccess;
    const KnnLayout ly(P);
    size_t sb = 0;
    cudaError_t e = sort_bytes(P, &sb);
    if (e != cudaSuccess) return e;
    uint32_t* bbox = reinterpret_cast<uint32_t*>(scratch + ly.bbox);
    uint64_t* keys_in = reinterpret_cast<uint64_t*>(scratch + ly.keys_in);
    uint64_t* keys_out = reinterpret_cast<uint64_t*>(scratch + ly.keys_out);
    uint32_t* idx_in = reinterpret_cast<uint32_t*>(scratch + ly.idx_in);
    uint32_t* idx_out = reinterpret_cast<uint32_t*>(scratch + ly.idx_out);
    float4* sorted = reinterpret_cast<float4*>(scratch + ly.pts);
    float4* lo = reinterpret_cast<float4*>(scratch + ly.box_lo);
    float4* hi = reinterpret_cast<float4*>(scratch + ly.box_hi);

    // min words start at the largest encoding, max words at the smallest
    if ((e = cudaMemsetAsync(bbox, 0xff, 3 * sizeof(uint32_t), s)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(bbox + 3, 0, 3 * sizeof(uint32_t), s)) != cudaSuccess) return e;
    bbox_kernel<<<std::min(blocks_for(P), 1024u), 256, 0, s>>>(P, points, bbox);
    morton_kernel<<<blocks_for(P), 256, 0, s>>>(P, points, bbox, keys_in, idx_in);
    g_launches += 2;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = cub::DeviceRadixSort::SortPairs(scratch + ly.sort_tmp, sb, keys_in, keys_out, idx_in, idx_out, P, 0, 63,
                                             s)) != cudaSuccess)
        return e;
    const KnnLevels& L = ly.lv;
    leaf_kernel<<<blocks_for((long long)L.count[0] * 32), 256, 0, s>>>(P, points, idx_out, sorted, lo, hi);
    g_launches++;
    for (int l = 1; l < L.n; l++) {
        node_kernel<<<blocks_for((long long)L.count[l] * 32), 256, 0, s>>>(L.count[l - 1], lo + L.off[l - 1],
                                                                          hi + L.off[l - 1], lo + L.off[l], hi + L.off[l]);
        g_launches++;
    }
    query_kernel<<<blocks_for((long long)L.count[0] * 32), 256, 0, s>>>(P, L.n - 1, L.off[L.n - 1], sorted, idx_out, lo,
                                                                        hi, out);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace f3dgs
