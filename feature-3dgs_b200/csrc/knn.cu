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
//
// Exact k-NN graph (launch_knn_graph, 1 <= k <= 32): steps 1-5 unchanged (build_tree), then graph_kernel, the same walk
// with a best-K list of (squared distance, input index) pairs per lane, K in {4, 8, 16, 32} the next size up from k, kept
// in registers by an unrolled compare-and-swap insertion.  Row i of idx / dist2 [P,k] is ascending by the pair
// (dist2, index) compared lexicographically, so ties go to the lower index; the point itself is excluded by index, and
// entries past P - 1 are (-1, +inf).  Exactness: a box is pruned only if its distance is ABOVE the current k-th distance
// (a box at exactly that distance may still hold a tie with a lower index).  By the argument above the box distance is
// a lower bound on the computed distance of every point inside, so each of them would come after the k-th pair.  The
// order of (distance, index) pairs is total, so the first k pairs are one set whatever the visiting order: results are
// bitwise reproducible, and a permutation of the input permutes the rows (and renames the indices) without changing
// dist2.  launch_knn_reverse builds the transpose in CSR form from idx with a stable radix sort of (neighbour, source).
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

// ---- exact k-NN graph: the same walk with a best-K list of (distance, index) pairs per lane

// (d, i) before (e, j) in a row of the graph: by distance, ties to the lower index (an empty slot, index 0xffffffff and
// +inf, comes after every point)
__device__ __forceinline__ bool pair_less(float d, uint32_t i, float e, uint32_t j) {
    return d < e || (d == e && i < j);
}

// The best pairs of one lane in K registers each for distances and indices (every index below is a compile-time
// constant).  For k < K the first K - k slots hold the sentinel (-inf, 0), which no pair comes before, so the k wanted
// pairs sit ascending in slots [K - k, K) and the last slot is the k-th.
template <int K>
struct BestK {
    float d[K];
    uint32_t i[K];
};

template <int K>
__device__ __forceinline__ void best_init(BestK<K>& b, int k) {
#pragma unroll
    for (int j = 0; j < K; j++) {
        b.d[j] = __int_as_float(j < K - k ? 0xff800000 : 0x7f800000);
        b.i[j] = j < K - k ? 0u : 0xffffffffu;
    }
}

// a pair before the k-th replaces it and sinks by one compare-and-swap per slot
template <int K>
__device__ __forceinline__ void best_insert(BestK<K>& b, float dv, uint32_t iv) {
    if (pair_less(dv, iv, b.d[K - 1], b.i[K - 1])) {
        b.d[K - 1] = dv;
        b.i[K - 1] = iv;
#pragma unroll
        for (int j = K - 1; j > 0; j--) {
            const float d0 = b.d[j - 1], d1 = b.d[j];
            const uint32_t i0 = b.i[j - 1], i1 = b.i[j];
            const bool sw = pair_less(d1, i1, d0, i0);
            b.d[j - 1] = sw ? d1 : d0;
            b.d[j] = sw ? d0 : d1;
            b.i[j - 1] = sw ? i1 : i0;
            b.i[j] = sw ? i0 : i1;
        }
    }
}

// best-K update of every lane against the points of one leaf; candidates carry their input index
template <int K>
__device__ __forceinline__ void scan_leaf_k(int P, long long leaf, const float4* __restrict__ sorted,
                                            const uint32_t* __restrict__ order, int lane, long long self, float3 q,
                                            bool active, BestK<K>& best) {
    const long long base = leaf * kLeaf;
    const int cnt = (int)min((long long)kLeaf, (long long)P - base);
    float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
    uint32_t ci = 0;
    if (lane < cnt) {
        c = sorted[base + lane];
        ci = order[base + lane];
    }
    for (int j = 0; j < cnt; j++) {
        const float cx = __shfl_sync(0xffffffffu, c.x, j);
        const float cy = __shfl_sync(0xffffffffu, c.y, j);
        const float cz = __shfl_sync(0xffffffffu, c.z, j);
        const uint32_t cj = __shfl_sync(0xffffffffu, ci, j);
        if (active && base + j != self) best_insert<K>(best, sq3(__fsub_rn(cx, q.x), __fsub_rn(cy, q.y), __fsub_rn(cz, q.z)), cj);
    }
}

template <int K>
__global__ void __launch_bounds__(256) graph_kernel(int P, int k, int top, long long top_off,
                                                    const float4* __restrict__ sorted, const uint32_t* __restrict__ order,
                                                    const float4* __restrict__ box_lo, const float4* __restrict__ box_hi,
                                                    int32_t* __restrict__ idx, float* __restrict__ dist2) {
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
    BestK<K> best;
    best_init<K>(best, k);
    scan_leaf_k<K>(P, leaf, sorted, order, lane, self, q, active, best);

    // query_kernel's walk; a box is entered unless its distance is above the k-th distance (a box at that distance can
    // still hold a tie with a lower index)
    int l = top;
    long long n = 0, off = top_off, cnt = 1;
    while (true) {
        const bool need = active && box_dist(q, box_lo[off + n], box_hi[off + n]) <= best.d[K - 1];
        if (__any_sync(0xffffffffu, need)) {
            if (l > 0) {
                l--;
                n *= kLeaf;
                cnt = level_count(P, l);
                off -= cnt;
                continue;
            }
            if (n != leaf) scan_leaf_k<K>(P, n, sorted, order, lane, self, q, active, best);
        }
        while (l < top && ((n & (kLeaf - 1)) == kLeaf - 1 || n + 1 >= cnt)) {
            off += cnt;
            l++;
            n >>= 5;
            cnt = level_count(P, l);
        }
        if (l == top) break;
        n++;
    }
    if (!active) return;
    const size_t row = (size_t)order[self] * k;
    const int skip = K - k;
#pragma unroll
    for (int j = 0; j < K; j++)
        if (j >= skip) {
            idx[row + j - skip] = (int32_t)best.i[j];
            dist2[row + j - skip] = best.d[j];
        }
}

// ---- reverse lists: a stable sort of the (neighbour, source) pairs by neighbour; -1 (or any index outside [0, P))
// sorts last as key P and is dropped
struct ReverseLayout {
    size_t keys_in, keys_out, vals_in, sort_tmp, fixed_bytes;
    explicit ReverseLayout(size_t E) {
        size_t o = 0;
        keys_in = o;   o = align_up(o + E * sizeof(uint32_t));
        keys_out = o;  o = align_up(o + E * sizeof(uint32_t));
        vals_in = o;   o = align_up(o + E * sizeof(int32_t));
        sort_tmp = o;
        fixed_bytes = o;
    }
};

int key_bits(int P) {  // keys are in [0, P]
    int b = 0;
    for (uint32_t n = (uint32_t)P; n; n >>= 1) b++;
    return b;
}

cudaError_t reverse_sort_bytes(int P, int k, size_t* bytes) {
    *bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                           (const int32_t*)nullptr, (int32_t*)nullptr, P * k, 0, key_bits(P));
}

__global__ void __launch_bounds__(256) reverse_keys_kernel(int P, int k, const int32_t* __restrict__ idx,
                                                           uint32_t* __restrict__ keys, int32_t* __restrict__ vals) {
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)P * k) return;
    const int32_t j = idx[e];
    keys[e] = (j >= 0 && j < P) ? (uint32_t)j : (uint32_t)P;
    vals[e] = (int32_t)(e / k);
}

// offsets[n] = the first sorted position whose key is >= n, for n in [0, P]; dropped entries become -1
__global__ void __launch_bounds__(256) reverse_offsets_kernel(int P, int E, const uint32_t* __restrict__ keys,
                                                              int32_t* __restrict__ sources, int32_t* __restrict__ offsets) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const uint32_t key = keys[e];
    const long long prev = e ? (long long)keys[e - 1] : -1;
    for (long long n = prev + 1; n <= key; n++) offsets[n] = e;
    if (e == E - 1)
        for (long long n = (long long)key + 1; n <= P; n++) offsets[n] = E;
    if (key == (uint32_t)P) sources[e] = -1;
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

namespace {

// Steps 1-5 of the pipeline, shared by every query: the sorted points, the Morton order idx_out and the boxes of every
// level, in `scratch` as laid out by `ly`
cudaError_t build_tree(int P, const float* points, char* scratch, const KnnLayout& ly, cudaStream_t s) {
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
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_knn_mean_dist(int P, const float* points, float* out, char* scratch, cudaStream_t s) {
    if (P <= 0) return cudaSuccess;
    const KnnLayout ly(P);
    cudaError_t e = build_tree(P, points, scratch, ly, s);
    if (e != cudaSuccess) return e;
    const KnnLevels& L = ly.lv;
    query_kernel<<<blocks_for((long long)L.count[0] * 32), 256, 0, s>>>(
        P, L.n - 1, L.off[L.n - 1], reinterpret_cast<const float4*>(scratch + ly.pts),
        reinterpret_cast<const uint32_t*>(scratch + ly.idx_out), reinterpret_cast<const float4*>(scratch + ly.box_lo),
        reinterpret_cast<const float4*>(scratch + ly.box_hi), out);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t knn_graph_scratch_bytes(int P, int k, size_t* bytes) {
    *bytes = 0;
    if (P <= 0) return cudaSuccess;
    size_t a = 0, b = 0;
    cudaError_t e = knn_scratch_bytes(P, &a);
    if (e != cudaSuccess) return e;
    if ((e = reverse_sort_bytes(P, k, &b)) != cudaSuccess) return e;
    *bytes = std::max(a, ReverseLayout((size_t)P * k).fixed_bytes + align_up(b));
    return cudaSuccess;
}

size_t knn_graph_scratch_fixed_bytes(int P, int k) {
    return P > 0 ? std::max(KnnLayout(P).fixed_bytes, ReverseLayout((size_t)P * k).fixed_bytes) : 0;
}

cudaError_t launch_knn_graph(int P, int k, const float* points, int32_t* idx, float* dist2, int32_t* order,
                             char* scratch, cudaStream_t s) {
    if (P <= 0) return cudaSuccess;
    const KnnLayout ly(P);
    cudaError_t e = build_tree(P, points, scratch, ly, s);
    if (e != cudaSuccess) return e;
    const KnnLevels& L = ly.lv;
    const float4* sorted = reinterpret_cast<const float4*>(scratch + ly.pts);
    const uint32_t* ord = reinterpret_cast<const uint32_t*>(scratch + ly.idx_out);
    const float4* lo = reinterpret_cast<const float4*>(scratch + ly.box_lo);
    const float4* hi = reinterpret_cast<const float4*>(scratch + ly.box_hi);
    const unsigned grid = blocks_for((long long)L.count[0] * 32);
    if (k <= 4)
        graph_kernel<4><<<grid, 256, 0, s>>>(P, k, L.n - 1, L.off[L.n - 1], sorted, ord, lo, hi, idx, dist2);
    else if (k <= 8)
        graph_kernel<8><<<grid, 256, 0, s>>>(P, k, L.n - 1, L.off[L.n - 1], sorted, ord, lo, hi, idx, dist2);
    else if (k <= 16)
        graph_kernel<16><<<grid, 256, 0, s>>>(P, k, L.n - 1, L.off[L.n - 1], sorted, ord, lo, hi, idx, dist2);
    else
        graph_kernel<32><<<grid, 256, 0, s>>>(P, k, L.n - 1, L.off[L.n - 1], sorted, ord, lo, hi, idx, dist2);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return cudaMemcpyAsync(order, ord, (size_t)P * sizeof(int32_t), cudaMemcpyDeviceToDevice, s);
}

cudaError_t launch_knn_reverse(int P, int k, const int32_t* idx, int32_t* offsets, int32_t* sources, char* scratch,
                               cudaStream_t s) {
    if (P <= 0) return cudaSuccess;
    const int E = P * k;
    const ReverseLayout ly((size_t)E);
    size_t sb = 0;
    cudaError_t e = reverse_sort_bytes(P, k, &sb);
    if (e != cudaSuccess) return e;
    uint32_t* keys_in = reinterpret_cast<uint32_t*>(scratch + ly.keys_in);
    uint32_t* keys_out = reinterpret_cast<uint32_t*>(scratch + ly.keys_out);
    int32_t* vals_in = reinterpret_cast<int32_t*>(scratch + ly.vals_in);
    reverse_keys_kernel<<<blocks_for(E), 256, 0, s>>>(P, k, idx, keys_in, vals_in);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // the radix sort is stable: each neighbour's sources stay in ascending row order
    if ((e = cub::DeviceRadixSort::SortPairs(scratch + ly.sort_tmp, sb, keys_in, keys_out, vals_in, sources, E, 0,
                                             key_bits(P), s)) != cudaSuccess)
        return e;
    reverse_offsets_kernel<<<blocks_for(E), 256, 0, s>>>(P, E, keys_out, sources, offsets);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace f3dgs
