// C-ABI entry points of libf3dgs_b200.so and the host-side orchestration of one view.
// Mirrors CudaRasterizer::Rasterizer::{forward,backward,markVisible}
// (reference rasterizer_impl.cu:198-342, :347-461, :141-153); see include/f3dgs_b200.h.
//
// Per forward call: 1 preprocess kernel, cub::DeviceScan::InclusiveSum, ONE 4-byte D2H copy +
// stream sync (num_rendered sizes the binning buffer and is returned to the caller, as in the
// reference rasterizer_impl.cu:283), key emission, cub::DeviceRadixSort::SortPairs on the
// minimal key width, range detection, composite.  Everything is enqueued on the caller's stream.
#include <cub/cub.cuh>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/f3dgs_b200.h"
#include "kernels.h"

namespace f3dgs {
std::atomic<unsigned long long> g_launches{0};
}
using namespace f3dgs;

namespace {

thread_local std::string t_error;

int fail(int code, const std::string& msg) {
    t_error = msg;
    return -code;
}

inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// ---- optional per-stage timing with CUDA events on the launch stream
struct StageRec {
    int stage;
    cudaEvent_t e0, e1;
};
bool g_profile = false;
std::mutex g_profile_mu;
std::vector<StageRec> g_recs;
std::vector<cudaEvent_t> g_event_pool;

cudaEvent_t get_event() {
    if (!g_event_pool.empty()) {
        cudaEvent_t e = g_event_pool.back();
        g_event_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
struct StageTimer {
    bool on;
    StageRec r;
    cudaStream_t s;
    StageTimer(int stage, cudaStream_t stream) : on(g_profile), s(stream) {
        if (!on) return;
        std::lock_guard<std::mutex> lk(g_profile_mu);
        r.stage = stage;
        r.e0 = get_event();
        r.e1 = get_event();
        cudaEventRecord(r.e0, s);
    }
    ~StageTimer() {
        if (!on) return;
        cudaEventRecord(r.e1, s);
        std::lock_guard<std::mutex> lk(g_profile_mu);
        g_recs.push_back(r);
    }
};

struct GeomLayout {
    size_t rec, cov3d, clamped, tiles, offsets, radii, fixed_bytes;
    explicit GeomLayout(size_t P) {
        size_t o = 0;
        rec = o;      o = align_up(o + P * sizeof(SplatRec));
        cov3d = o;    o = align_up(o + P * 6 * sizeof(float));
        clamped = o;  o = align_up(o + P);
        tiles = o;    o = align_up(o + P * 4);
        offsets = o;  o = align_up(o + P * 4);
        radii = o;    o = align_up(o + P * 4);
        fixed_bytes = o;
    }
};
struct ImgLayout {
    size_t final_T, n_contrib, ranges, counters, bytes;
    ImgLayout(size_t HW, size_t tiles) {
        size_t o = 0;
        final_T = o;    o = align_up(o + HW * 4);
        n_contrib = o;  o = align_up(o + HW * 4);
        ranges = o;     o = align_up(o + tiles * 8);
        counters = o;   o = align_up(o + 256);  // tile work counters of the persistent composite kernels
        bytes = o;
    }
};
struct BinLayout {
    size_t point_list, keys, point_list_unsorted, keys_unsorted, fixed_bytes;
    explicit BinLayout(size_t R) {
        size_t o = 0;
        point_list = o;           o = align_up(o + R * 4);
        keys = o;                 o = align_up(o + R * 8);
        point_list_unsorted = o;  o = align_up(o + R * 4);
        keys_unsorted = o;        o = align_up(o + R * 8);
        fixed_bytes = o;
    }
};

// Per (tile, 8x4 block) instance lists of the two-kernel backward: 8R entries of capacity (block b of a tile owns `len` of them).
struct ListLayout {
    size_t w, meta, cnt, bytes;
    ListLayout(size_t R, size_t tiles) {
        size_t o = 0;
        w = o;     o = align_up(o + 8 * R * 32 * sizeof(float));
        meta = o;  o = align_up(o + 8 * R * sizeof(uint2));
        cnt = o;   o = align_up(o + 8 * tiles * sizeof(uint32_t));
        bytes = o;
    }
};

inline int bit_length(uint32_t n) {
    int b = 0;
    while (n) {
        b++;
        n >>= 1;
    }
    return b;
}

#define CUDA_TRY(expr)                                                                              \
    do {                                                                                            \
        cudaError_t e_ = (expr);                                                                    \
        if (e_ != cudaSuccess)                                                                      \
            return fail(F3DGS_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));        \
    } while (0)

// reference CHECK_CUDA (auxiliary.h:172-179): in debug mode synchronise and surface errors per stage
#define STAGE_CHECK(name)                                                                           \
    do {                                                                                            \
        cudaError_t e_ = cudaGetLastError();                                                        \
        if (e_ == cudaSuccess && debug) e_ = cudaStreamSynchronize(stream);                         \
        if (e_ != cudaSuccess)                                                                      \
            return fail(F3DGS_ERR_CUDA, std::string("stage ") + name + ": " + cudaGetErrorString(e_)); \
    } while (0)

ViewParams make_view(int P, int D, int M, int C, int width, int height, float tan_fovx, float tan_fovy,
                     float scale_modifier, const float* viewmatrix, const float* projmatrix,
                     const float* cam_pos) {
    ViewParams vp;
    vp.P = P; vp.D = D; vp.M = M; vp.C = C; vp.W = width; vp.H = height;
    vp.grid_x = (uint32_t)((width + F3DGS_TILE - 1) / F3DGS_TILE);
    vp.grid_y = (uint32_t)((height + F3DGS_TILE - 1) / F3DGS_TILE);
    vp.tan_fovx = tan_fovx; vp.tan_fovy = tan_fovy;
    vp.focal_y = height / (2.0f * tan_fovy);  // reference rasterizer_impl.cu:225-226
    vp.focal_x = width / (2.0f * tan_fovx);
    vp.scale_modifier = scale_modifier;
    vp.viewmatrix = viewmatrix; vp.projmatrix = projmatrix; vp.cam_pos = cam_pos;
    return vp;
}

}  // namespace

extern "C" {

int f3dgs_abi_version(void) { return F3DGS_ABI_VERSION; }
const char* f3dgs_last_error(void) { return t_error.c_str(); }
unsigned long long f3dgs_launch_count(void) { return g_launches.load(); }

void f3dgs_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(g_profile_mu);
    g_profile = on != 0;
}

int f3dgs_profile_read(double* ms, unsigned long long* count) {
    if (!ms || !count) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_profile_read: NULL output");
    std::lock_guard<std::mutex> lk(g_profile_mu);
    for (const StageRec& r : g_recs) {
        float t = 0.f;
        cudaError_t e = cudaEventSynchronize(r.e1);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&t, r.e0, r.e1);
        if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("profile_read: ") + cudaGetErrorString(e));
        if (r.stage >= 0 && r.stage < F3DGS_N_STAGES) {
            ms[r.stage] += t;
            count[r.stage] += 1;
        }
        g_event_pool.push_back(r.e0);
        g_event_pool.push_back(r.e1);
    }
    g_recs.clear();
    return 0;
}

int f3dgs_get_layout(int P, int width, int height, int R, f3dgs_layout* out) {
    if (!out || P < 0 || width <= 0 || height <= 0 || R < 0)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_get_layout: bad argument");
    const GeomLayout g((size_t)P);
    const size_t tiles = (size_t)((width + 15) / 16) * ((height + 15) / 16);
    const ImgLayout im((size_t)width * height, tiles);
    const BinLayout b((size_t)R);
    out->geom_bytes = g.fixed_bytes; out->geom_rec = g.rec; out->geom_cov3d = g.cov3d;
    out->geom_clamped = g.clamped; out->geom_tiles = g.tiles; out->geom_offsets = g.offsets;
    out->geom_radii = g.radii;
    out->img_bytes = im.bytes; out->img_final_T = im.final_T; out->img_n_contrib = im.n_contrib;
    out->img_ranges = im.ranges;
    out->bin_bytes = b.fixed_bytes; out->bin_point_list = b.point_list; out->bin_keys = b.keys;
    return 0;
}

int f3dgs_forward(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx, f3dgs_alloc_fn binning_alloc,
                  void* binning_ctx, f3dgs_alloc_fn image_alloc, void* image_ctx, int P, int D, int M, int C,
                  const float* background, int width, int height, const float* means3D, const float* shs,
                  const float* colors_precomp, const float* semantic_feature, const float* opacities,
                  const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
                  const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                  float tan_fovy, int prefiltered, float* out_color, float* out_feature_map, float* out_depth,
                  int* radii, int debug, void* cuda_stream) {
    t_error.clear();
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (P < 0 || width <= 0 || height <= 0 || C < 0 || C > F3DGS_MAX_FEATURE_DIM || D < 0 || D > 3)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_forward: bad sizes (P, width, height, C or D)");
    if (!geometry_alloc || !binning_alloc || !image_alloc)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_forward: missing allocator");
    if (P == 0) return 0;
    if (!means3D || !opacities || !background || !viewmatrix || !projmatrix || !cam_pos || !out_color ||
        !out_depth)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_forward: NULL required pointer");
    if ((shs == nullptr) == (colors_precomp == nullptr))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_forward: provide exactly one of shs / colors_precomp");
    if (((scales == nullptr) || (rotations == nullptr)) == (cov3D_precomp == nullptr))
        return fail(F3DGS_ERR_INVALID_ARGUMENT,
                    "f3dgs_forward: provide exactly one of (scales, rotations) / cov3D_precomp");
    if (C > 0 && (!semantic_feature || !out_feature_map))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_forward: C > 0 needs semantic_feature and out_feature_map");
    if (shs && M < (D + 1) * (D + 1))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_forward: M < (D+1)^2 SH coefficients");

    const ViewParams vp = make_view(P, D, M, C, width, height, tan_fovx, tan_fovy, scale_modifier, viewmatrix,
                                    projmatrix, cam_pos);
    const size_t tiles = (size_t)vp.grid_x * vp.grid_y;

    // ---- geometry buffer
    const GeomLayout gl((size_t)P);
    size_t scan_bytes = 0;
    CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, P, stream));
    char* geom = geometry_alloc(geometry_ctx, gl.fixed_bytes + align_up(scan_bytes));
    if (!geom) return fail(F3DGS_ERR_ALLOC, "geometry allocator returned NULL");
    SplatRec* rec = reinterpret_cast<SplatRec*>(geom + gl.rec);
    float* cov3d = reinterpret_cast<float*>(geom + gl.cov3d);
    uint8_t* clamped = reinterpret_cast<uint8_t*>(geom + gl.clamped);
    uint32_t* tiles_touched = reinterpret_cast<uint32_t*>(geom + gl.tiles);
    uint32_t* offsets = reinterpret_cast<uint32_t*>(geom + gl.offsets);
    int* radii_int = reinterpret_cast<int*>(geom + gl.radii);
    if (radii == nullptr) radii = radii_int;  // reference rasterizer_impl.cu:232-235

    // ---- image buffer
    const ImgLayout il((size_t)width * height, tiles);
    char* img = image_alloc(image_ctx, il.bytes);
    if (!img) return fail(F3DGS_ERR_ALLOC, "image allocator returned NULL");
    float* final_T = reinterpret_cast<float*>(img + il.final_T);
    uint32_t* n_contrib = reinterpret_cast<uint32_t*>(img + il.n_contrib);
    uint2* ranges = reinterpret_cast<uint2*>(img + il.ranges);

    {
        StageTimer t(F3DGS_STAGE_PREPROCESS_FWD, stream);
        launch_preprocess_fwd(vp, means3D, scales, rotations, opacities, shs, cov3D_precomp, colors_precomp,
                              prefiltered != 0, radii, rec, cov3d, clamped, tiles_touched, stream);
    }
    STAGE_CHECK("preprocess");
    {
        StageTimer t(F3DGS_STAGE_SCAN, stream);
        CUDA_TRY(cub::DeviceScan::InclusiveSum(geom + gl.fixed_bytes, scan_bytes, tiles_touched, offsets, P, stream));
    }
    STAGE_CHECK("scan");

    // one pinned word per calling thread for the 4-byte read-back; released when the thread ends
    struct PinnedInt {
        int* p = nullptr;
        ~PinnedInt() {
            if (p) cudaFreeHost(p);
        }
    };
    static thread_local PinnedInt pinned;
    if (!pinned.p) CUDA_TRY(cudaHostAlloc((void**)&pinned.p, sizeof(int), cudaHostAllocDefault));
    int* h_count = pinned.p;
    CUDA_TRY(cudaMemcpyAsync(h_count, offsets + (P - 1), sizeof(int), cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    const int R = *h_count;
    if (R < 0) return fail(F3DGS_ERR_CUDA, "num_rendered overflowed int32");

    // ---- binning buffer
    const BinLayout bl((size_t)R);
    const int end_bit = 32 + bit_length((uint32_t)(tiles > 0 ? tiles - 1 : 0));
    size_t sort_bytes = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr,
                                             (uint32_t*)nullptr, (uint32_t*)nullptr, R, 0, end_bit, stream));
    char* bin = binning_alloc(binning_ctx, bl.fixed_bytes + align_up(sort_bytes));
    if (!bin) return fail(F3DGS_ERR_ALLOC, "binning allocator returned NULL");
    uint32_t* point_list = reinterpret_cast<uint32_t*>(bin + bl.point_list);
    uint64_t* keys = reinterpret_cast<uint64_t*>(bin + bl.keys);
    uint32_t* point_list_unsorted = reinterpret_cast<uint32_t*>(bin + bl.point_list_unsorted);
    uint64_t* keys_unsorted = reinterpret_cast<uint64_t*>(bin + bl.keys_unsorted);

    CUDA_TRY(cudaMemsetAsync(ranges, 0, tiles * sizeof(uint2), stream));
    if (R > 0) {
        {
            StageTimer t(F3DGS_STAGE_DUPLICATE_KEYS, stream);
            launch_duplicate_keys(P, rec, offsets, radii, vp.grid_x, vp.grid_y, keys_unsorted, point_list_unsorted,
                                  stream);
        }
        STAGE_CHECK("duplicate_keys");
        {
            StageTimer t(F3DGS_STAGE_SORT, stream);
            CUDA_TRY(cub::DeviceRadixSort::SortPairs(bin + bl.fixed_bytes, sort_bytes, keys_unsorted, keys,
                                                     point_list_unsorted, point_list, R, 0, end_bit, stream));
        }
        STAGE_CHECK("sort");
        {
            StageTimer t(F3DGS_STAGE_TILE_RANGES, stream);
            launch_tile_ranges(R, keys, ranges, stream);
        }
        STAGE_CHECK("tile_ranges");
    }

    cudaError_t e;
    {
        StageTimer t(F3DGS_STAGE_COMPOSITE_FWD, stream);
        int* counters = reinterpret_cast<int*>(img + il.counters);
        e = launch_composite_fwd(vp, ranges, point_list, rec, semantic_feature, background, final_T, n_contrib,
                                 out_color, out_feature_map, out_depth, counters, stream);
    }
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("composite_fwd launch: ") + cudaGetErrorString(e));
    STAGE_CHECK("composite_fwd");
    return R;
}

}  // extern "C"

namespace {

struct ScratchLayout {  // per-view intermediates of the accumulating backward (all zeroed per call)
    size_t mean2D, conic, dz, color, cov3D, bytes;
    explicit ScratchLayout(size_t P) {
        size_t o = 0;
        mean2D = o;  o = align_up(o + P * 3 * 4);
        conic = o;   o = align_up(o + P * 4 * 4);
        dz = o;      o = align_up(o + P * 4);
        color = o;   o = align_up(o + P * 3 * 4);
        cov3D = o;   o = align_up(o + P * 6 * 4);
        bytes = o;
    }
};

// Shared body of f3dgs_backward (accumulate = false: the reference's assign-into-zeroed-buffers contract) and
// f3dgs_backward_accum (accumulate = true: += into the caller's per-parameter gradient buffers).
int backward_impl(const char* who, bool accumulate, int P, int D, int M, int R, int C, const float* background, int width,
                  int height, const float* means3D, const float* shs, const float* scales, float scale_modifier,
                  const float* rotations, const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                  const float* cam_pos, float tan_fovx, float tan_fovy, const int* radii, char* geom_buffer,
                  char* binning_buffer, char* image_buffer, const float* dL_dpix, const float* dL_dfeaturepix,
                  const float* dL_depths, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                  float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale,
                  float* dL_drot, float* dL_dz, float* grad_accum, float* denom, cudaEvent_t composite_done, int debug,
                  cudaStream_t stream) {
    const std::string w(who);
    if (P < 0 || width <= 0 || height <= 0 || C < 0 || C > F3DGS_MAX_FEATURE_DIM || R < 0)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, w + ": bad sizes");
    if (P == 0) return 0;
    if (!geom_buffer || !binning_buffer || !image_buffer)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, w + ": missing forward buffers");
    if (!dL_dpix || !dL_depths || (C > 0 && (!dL_dfeaturepix || !dL_dsemantic_feature)) || !dL_dmean2D ||
        !dL_dconic || !dL_dopacity || !dL_dcolor || !dL_dmean3D || !dL_dcov3D || !dL_dz)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, w + ": NULL gradient pointer");
    if (shs && !dL_dsh) return fail(F3DGS_ERR_INVALID_ARGUMENT, w + ": shs given but dL_dsh NULL");
    if (scales && (!rotations || !dL_dscale || !dL_drot))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, w + ": scales given but rotations/dL_dscale/dL_drot NULL");
    if ((grad_accum == nullptr) != (denom == nullptr))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, w + ": grad_accum and denom go together");

    const ViewParams vp = make_view(P, D, M, C, width, height, tan_fovx, tan_fovy, scale_modifier, viewmatrix,
                                    projmatrix, cam_pos);
    const size_t tiles = (size_t)vp.grid_x * vp.grid_y;
    const GeomLayout gl((size_t)P);
    const ImgLayout il((size_t)width * height, tiles);
    const BinLayout bl((size_t)R);
    const SplatRec* rec = reinterpret_cast<const SplatRec*>(geom_buffer + gl.rec);
    const float* cov3d = cov3D_precomp ? cov3D_precomp : reinterpret_cast<const float*>(geom_buffer + gl.cov3d);
    const uint8_t* clamped = reinterpret_cast<const uint8_t*>(geom_buffer + gl.clamped);
    if (radii == nullptr) radii = reinterpret_cast<const int*>(geom_buffer + gl.radii);
    const float* final_T = reinterpret_cast<const float*>(image_buffer + il.final_T);
    const uint32_t* n_contrib = reinterpret_cast<const uint32_t*>(image_buffer + il.n_contrib);
    const uint2* ranges = reinterpret_cast<const uint2*>(image_buffer + il.ranges);
    const uint32_t* point_list = reinterpret_cast<const uint32_t*>(binning_buffer + bl.point_list);

    cudaError_t e;
    {
        StageTimer t(F3DGS_STAGE_COMPOSITE_BWD, stream);
        int* counters = reinterpret_cast<int*>(image_buffer + il.counters);
        // Two kernels: the geometric gradients come from the alpha-only kernel at two CTAs per SM, which also emits the
        // blend weights per (tile, block) when there are features; the feature gradient is a second, streaming kernel
        // over those lists (feature_bwd.cu).
        char* lists = nullptr;
        const ListLayout ll((size_t)R, tiles);
        if (C > 0 && R > 0) {
            // stream-ordered scratch (the reference's backward allocates its scratch too, rasterizer_impl.cu:402-430);
            // the default pool keeps freed blocks, so steady-state calls do not reach the driver
            static std::once_flag once;
            std::call_once(once, [] {
                int dev = 0;
                cudaGetDevice(&dev);
                cudaMemPool_t pool;
                if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
                    unsigned long long keep = ~0ull;
                    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
                }
            });
            cudaError_t ea = cudaMallocAsync((void**)&lists, ll.bytes, stream);
            if (ea != cudaSuccess)
                return fail(F3DGS_ERR_ALLOC, w + ": cudaMallocAsync of " + std::to_string(ll.bytes) +
                                                 " bytes for the backward instance lists failed: " +
                                                 cudaGetErrorString(ea));
        }
        e = launch_composite_bwd_geom(
            vp, ranges, point_list, rec, background, final_T, n_contrib, dL_dpix, dL_depths, dL_dmean2D, dL_dconic,
            dL_dopacity, dL_dcolor, dL_dz, counters + 16, stream, lists ? reinterpret_cast<float*>(lists + ll.w) : nullptr,
            lists ? reinterpret_cast<uint2*>(lists + ll.meta) : nullptr,
            lists ? reinterpret_cast<uint32_t*>(lists + ll.cnt) : nullptr);
        if (e == cudaSuccess && lists)
            e = launch_feature_bwd(vp, ranges, reinterpret_cast<const float*>(lists + ll.w),
                                   reinterpret_cast<const uint2*>(lists + ll.meta),
                                   reinterpret_cast<const uint32_t*>(lists + ll.cnt), dL_dfeaturepix,
                                   dL_dsemantic_feature, counters + 48, stream);
        if (lists) cudaFreeAsync(lists, stream);
    }
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("composite_bwd launch: ") + cudaGetErrorString(e));
    STAGE_CHECK("composite_bwd");
    if (composite_done) CUDA_TRY(cudaEventRecord(composite_done, stream));
    {
        StageTimer t(F3DGS_STAGE_PREPROCESS_BWD, stream);
        launch_preprocess_bwd(vp, means3D, radii, shs, clamped, scales, rotations, cov3d, dL_dmean2D, dL_dconic,
                              dL_dmean3D, dL_dcolor, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dz, stream, accumulate,
                              grad_accum, denom);
    }
    STAGE_CHECK("preprocess_bwd");
    return 0;
}

}  // namespace

extern "C" {

int f3dgs_backward(int P, int D, int M, int R, int C, const float* background, int width, int height,
                   const float* means3D, const float* shs, const float* colors_precomp,
                   const float* semantic_feature, const float* scales, float scale_modifier,
                   const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                   const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
                   const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                   const float* dL_dpix, const float* dL_dfeaturepix, const float* dL_depths, float* dL_dmean2D,
                   float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dsemantic_feature,
                   float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                   float* dL_dz, int debug, void* cuda_stream) {
    (void)semantic_feature;  // not needed: dL/dfeature depends only on the blend weights (SURVEY D.1/D.2)
    (void)colors_precomp;    // colours were copied into the per-Gaussian records by the forward
    t_error.clear();
    return backward_impl("f3dgs_backward", false, P, D, M, R, C, background, width, height, means3D, shs, scales,
                         scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy,
                         radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, dL_dfeaturepix, dL_depths, dL_dmean2D,
                         dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
                         dL_drot, dL_dz, nullptr, nullptr, nullptr, debug, (cudaStream_t)cuda_stream);
}

size_t f3dgs_backward_scratch_bytes(int P) { return P > 0 ? ScratchLayout((size_t)P).bytes : 0; }

int f3dgs_backward_accum(int P, int D, int M, int R, int C, const float* background, int width, int height,
                         const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                         float scale_modifier, const float* rotations, const float* cov3D_precomp,
                         const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                         float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                         const float* dL_dpix, const float* dL_dfeaturepix, const float* dL_depths, char* scratch,
                         float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature, float* dL_dmean3D,
                         float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale, float* dL_drot,
                         float* dL_dmean2D_out, float* grad_accum, float* denom, void* composite_done_event, int debug,
                         void* cuda_stream) {
    t_error.clear();
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (P <= 0) return P == 0 ? 0 : fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_backward_accum: bad sizes");
    if (!scratch) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_backward_accum: NULL scratch");
    if ((colors_precomp != nullptr) != (dL_dcolors_precomp != nullptr) ||
        (cov3D_precomp != nullptr) != (dL_dcov3D_precomp != nullptr))
        return fail(F3DGS_ERR_INVALID_ARGUMENT,
                    "f3dgs_backward_accum: dL_dcolors_precomp / dL_dcov3D_precomp go with colors_precomp / cov3D_precomp");
    const ScratchLayout sl((size_t)P);
    CUDA_TRY(cudaMemsetAsync(scratch, 0, sl.bytes, stream));
    float* m2d = reinterpret_cast<float*>(scratch + sl.mean2D);
    // colours / cov3D are intermediates unless they are inputs of the caller (then their gradients accumulate)
    float* dcol = dL_dcolors_precomp ? dL_dcolors_precomp : reinterpret_cast<float*>(scratch + sl.color);
    float* dcov = dL_dcov3D_precomp ? dL_dcov3D_precomp : reinterpret_cast<float*>(scratch + sl.cov3D);
    const int rc = backward_impl(
        "f3dgs_backward_accum", true, P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier,
        rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
        binning_buffer, image_buffer, dL_dpix, dL_dfeaturepix, dL_depths, m2d,
        reinterpret_cast<float*>(scratch + sl.conic), dL_dopacity, dcol, dL_dsemantic_feature, dL_dmean3D, dcov, dL_dsh,
        dL_dscale, dL_drot, reinterpret_cast<float*>(scratch + sl.dz), grad_accum, denom,
        (cudaEvent_t)composite_done_event, debug, stream);
    if (rc < 0) return rc;
    if (dL_dmean2D_out)
        CUDA_TRY(cudaMemcpyAsync(dL_dmean2D_out, m2d, (size_t)P * 3 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    return 0;
}

}  // extern "C"

namespace {
bool ranges_overlap(const void* a, size_t na, const void* b, size_t nb) {
    if (!a || !b) return false;
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + nb && y < x + na;
}

// The float16 entry points (_f16gt, _f16) validate and launch as their float32 twins do; `fn` is the twin's name without
// the f3dgs_ prefix.  Half data is IEEE binary16 bits at the ABI (uint16_t) and __half in the kernels.
template <typename GT>
int feature_resize_fwd_impl(const char* fn, int C, int H, int W, int Hg, int Wg, const float* feature_map, const GT* gt,
                            float grad_scale, float* out, float* loss_sum, void* cuda_stream) {
    const std::string api = std::string("f3dgs_") + fn;
    t_error.clear();
    if (C < 0 || H <= 0 || W <= 0 || Hg <= 0 || Wg <= 0) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": bad sizes");
    if (C == 0) return 0;
    if (!feature_map || !out) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": NULL pointer");
    if constexpr (std::is_same_v<GT, __half>) {
        // no target is the float32 symbol's job; out's 4-byte elements cannot alias gt's 2-byte ones element for element
        if (!gt) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": NULL pointer (gt is required)");
        const size_t n = (size_t)C * Hg * Wg;
        if (ranges_overlap(out, n * 4, feature_map, (size_t)C * H * W * 4) || ranges_overlap(out, n * 4, gt, n * 2))
            return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": out overlaps feature_map or gt");
    }
    cudaError_t e = launch_feature_resize_fwd(C, H, W, Hg, Wg, feature_map, gt, grad_scale, out, loss_sum,
                                              (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
    return 0;
}
}  // namespace

extern "C" {

int f3dgs_feature_resize_fwd(int C, int H, int W, int Hg, int Wg, const float* feature_map, const float* gt,
                             float grad_scale, float* out, float* loss_sum, void* cuda_stream) {
    return feature_resize_fwd_impl("feature_resize_fwd", C, H, W, Hg, Wg, feature_map, gt, grad_scale, out, loss_sum,
                                   cuda_stream);
}

int f3dgs_feature_resize_fwd_f16gt(int C, int H, int W, int Hg, int Wg, const float* feature_map, const uint16_t* gt,
                                   float grad_scale, float* out, float* loss_sum, void* cuda_stream) {
    return feature_resize_fwd_impl("feature_resize_fwd_f16gt", C, H, W, Hg, Wg, feature_map,
                                   reinterpret_cast<const __half*>(gt), grad_scale, out, loss_sum, cuda_stream);
}

int f3dgs_feature_resize_bwd(int C, int H, int W, int Hg, int Wg, const float* dout, float* dL_dfeature_map,
                             void* cuda_stream) {
    t_error.clear();
    if (C < 0 || H <= 0 || W <= 0 || Hg <= 0 || Wg <= 0)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_feature_resize_bwd: bad sizes");
    if (C == 0) return 0;
    if (!dout || !dL_dfeature_map) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_feature_resize_bwd: NULL pointer");
    cudaError_t e = launch_feature_resize_bwd(C, H, W, Hg, Wg, dout, dL_dfeature_map, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("feature_resize_bwd: ") + cudaGetErrorString(e));
    return 0;
}

int f3dgs_image_loss(int planes, int H, int W, const float* image, const float* gt, float w_l1, float w_ssim, float* sums,
                     float* dL_dimage, void* cuda_stream) {
    t_error.clear();
    if (planes < 0 || H <= 0 || W <= 0) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_image_loss: bad sizes");
    if (planes == 0) return 0;
    if (!image_loss_grid_ok(planes, H, W))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_image_loss: sizes exceed the launch grid limits");
    if (!image || !gt || !sums) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_image_loss: NULL pointer");
    if (dL_dimage) {  // a CTA reads its neighbours' pixels (the window halo), so the gradient cannot overwrite an input
        const uintptr_t n = (uintptr_t)planes * H * W * sizeof(float), d = (uintptr_t)dL_dimage;
        auto overlaps = [&](const float* p) { return d < (uintptr_t)p + n && (uintptr_t)p < d + n; };
        if (overlaps(image) || overlaps(gt))
            return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_image_loss: dL_dimage overlaps image or gt");
    }
    cudaError_t e = launch_image_loss(planes, H, W, image, gt, w_l1, w_ssim, sums, dL_dimage, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("image_loss: ") + cudaGetErrorString(e));
    return 0;
}

}  // extern "C"

namespace {
template <typename Y>
int decoder_forward_impl(const char* fn, int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                         Y* y, void* cuda_stream) {
    const std::string api = std::string("f3dgs_") + fn;
    t_error.clear();
    if (Cin < 1 || Cin > kDecoderMaxCin || Cout < 1 || Cout > kDecoderMaxCout || N < 1)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": bad sizes (1 <= Cin <= 256, 1 <= Cout <= 4096, N >= 1)");
    if (!decoder_grid_ok(Cin, Cout, N))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": sizes exceed the launch grid limits");
    if (!weight || !x || !y) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": NULL pointer");
    const size_t ny = (size_t)Cout * N * sizeof(Y);
    if (ranges_overlap(y, ny, weight, (size_t)Cout * Cin * 4) || ranges_overlap(y, ny, bias, (size_t)Cout * 4) ||
        ranges_overlap(y, ny, x, (size_t)Cin * N * 4))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": y overlaps an input");
    cudaError_t e = launch_decoder_forward(Cin, Cout, N, weight, bias, x, y, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
    return 0;
}

template <typename GT>
int decoder_l1_impl(const char* fn, int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                    const GT* gt, float grad_scale, float* loss_sum, float* dL_dx, float* dL_dweight, float* dL_dbias,
                    void* cuda_stream) {
    const std::string api = std::string("f3dgs_") + fn;
    t_error.clear();
    if (Cin < 1 || Cin > kDecoderMaxCin || Cout < 1 || Cout > kDecoderMaxCout || N < 1)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": bad sizes (1 <= Cin <= 256, 1 <= Cout <= 4096, N >= 1)");
    if (!decoder_grid_ok(Cin, Cout, N))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": sizes exceed the launch grid limits");
    if (!weight || !x || !gt || !loss_sum || !dL_dx || !dL_dweight)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": NULL pointer");
    if ((bias == nullptr) != (dL_dbias == nullptr))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": NULL pointer (dL_dbias goes with bias)");
    const size_t nx = (size_t)Cin * N * 4, nw = (size_t)Cout * Cin * 4, nb = (size_t)Cout * 4;
    // a warp reads x of its own pixels only, but kernel B reads all of x after dL_dx is written
    if (ranges_overlap(dL_dx, nx, x, nx) || ranges_overlap(dL_dx, nx, gt, (size_t)Cout * N * sizeof(GT)) ||
        ranges_overlap(dL_dx, nx, weight, nw) || ranges_overlap(dL_dx, nx, bias, nb) ||
        ranges_overlap(dL_dx, nx, dL_dweight, nw) || ranges_overlap(dL_dx, nx, dL_dbias, nb))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": dL_dx overlaps an input");
    cudaError_t e = launch_decoder_l1(Cin, Cout, N, weight, bias, x, gt, grad_scale, loss_sum, dL_dx, dL_dweight,
                                      dL_dbias, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
    return 0;
}

template <typename X>
int feature_query_impl(const char* fn, int C, int D, int K, int N, const float* weight, const float* bias, const X* x,
                       const float* text, float logit_scale, const uint8_t* positive, int64_t* labels, float* prob,
                       float* logits, void* cuda_stream) {
    const std::string api = std::string("f3dgs_") + fn;
    t_error.clear();
    if (K < 1 || K > kQueryMaxK || D < 1 || D > kQueryMaxD || C < 1 || N < 0 || (weight && C > kDecoderMaxCin))
        return fail(F3DGS_ERR_INVALID_ARGUMENT,
                    api + ": bad sizes (1 <= K <= 256, 1 <= D <= 4096, N >= 0, 1 <= C <= 256 with a decoder)");
    if (!weight && D != C) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": D != C needs a decoder weight");
    if (bias && !weight) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": bias without weight");
    if (!x || !text) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": NULL pointer (x and text are required)");
    if (!labels && !prob && !logits) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": no output requested");
    if (prob && !positive) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": prob needs a positive set");
    if (!std::isfinite(logit_scale)) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": logit_scale is not finite");
    const size_t n = (size_t)N;
    struct Range {
        const void* p;
        size_t bytes;
    };
    const Range in[] = {{weight, (size_t)D * C * 4}, {bias, (size_t)D * 4}, {x, (size_t)C * n * sizeof(X)},
                        {text, (size_t)K * D * 4}, {positive, (size_t)K}};
    const Range out[] = {{labels, n * 8}, {prob, n * 4}, {logits, (size_t)K * n * 4}};
    for (int i = 0; i < 3; i++) {
        for (const Range& r : in)
            if (ranges_overlap(out[i].p, out[i].bytes, r.p, r.bytes))
                return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": an output overlaps an input");
        for (int j = 0; j < i; j++)
            if (ranges_overlap(out[i].p, out[i].bytes, out[j].p, out[j].bytes))
                return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": outputs overlap");
    }
    cudaError_t e = launch_feature_query(C, D, K, N, weight, bias, x, text, logit_scale, positive, labels, prob, logits,
                                         (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
    return 0;
}

// ---- feature PCA: shared validation of (C, N) and of output ranges against inputs
bool pca_sizes_ok(int C, int N) { return C >= kPcaMinC && C <= kPcaMaxC && N >= 7; }  // n = ceil(N / 3) >= 3

struct Range {
    const void* p;
    size_t bytes;
};
bool any_overlap(const Range& out, std::initializer_list<Range> in) {
    for (const Range& r : in)
        if (ranges_overlap(out.p, out.bytes, r.p, r.bytes)) return true;
    return false;
}

template <typename X>
int pca_moments_impl(const char* fn, int C, int N, const X* x, char* scratch, float* mean, double* cov,
                     void* cuda_stream) {
    const std::string api = std::string("f3dgs_") + fn;
    t_error.clear();
    if (!pca_sizes_ok(C, N)) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": bad sizes (3 <= C <= 1024, N >= 7)");
    if (!x || !scratch || !mean || !cov) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": NULL pointer");
    const Range rx{x, (size_t)C * N * sizeof(X)}, rs{scratch, pca_scratch_fixed_bytes(C, N)};
    const Range rm{mean, (size_t)C * 4}, rc{cov, (size_t)C * C * 8};
    if (any_overlap(rs, {rx}) || any_overlap(rm, {rx, rs}) || any_overlap(rc, {rx, rs, rm}))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": scratch, mean and cov must not overlap x or each other");
    cudaError_t e = launch_pca_moments(C, N, x, scratch, mean, cov, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
    return 0;
}

template <typename X>
int pca_range_impl(const char* fn, int C, int N, const X* x, const float* mean, const float* components, char* scratch,
                   float* range, void* cuda_stream) {
    const std::string api = std::string("f3dgs_") + fn;
    t_error.clear();
    if (!pca_sizes_ok(C, N)) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": bad sizes (3 <= C <= 1024, N >= 7)");
    if (!x || !mean || !components || !scratch || !range) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": NULL pointer");
    const Range rx{x, (size_t)C * N * sizeof(X)}, rm{mean, (size_t)C * 4}, rc{components, (size_t)3 * C * 4};
    const Range rs{scratch, pca_scratch_fixed_bytes(C, N)}, rr{range, 8};
    if (any_overlap(rs, {rx, rm, rc}) || any_overlap(rr, {rx, rm, rc, rs}))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": scratch or range overlaps an input");
    size_t sb = 0;
    CUDA_TRY(pca_scratch_bytes(C, N, &sb));  // the sort's share of the scratch is sized by CUB for the current device
    if (any_overlap({scratch, sb}, {rx, rm, rc, rr}))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": scratch or range overlaps an input");
    cudaError_t e = launch_pca_range(C, N, x, mean, components, scratch, range, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
    return 0;
}

template <typename X>
int pca_image_impl(const char* fn, int C, int N, const X* x, const float* mean, const float* components,
                   const float* range, float* image, void* cuda_stream) {
    const std::string api = std::string("f3dgs_") + fn;
    t_error.clear();
    if (!pca_sizes_ok(C, N)) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": bad sizes (3 <= C <= 1024, N >= 7)");
    if (!x || !mean || !components || !range || !image) return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": NULL pointer");
    const Range ri{image, (size_t)N * 3 * 4};
    if (any_overlap(ri, {{x, (size_t)C * N * sizeof(X)}, {mean, (size_t)C * 4}, {components, (size_t)3 * C * 4},
                         {range, 8}}))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, api + ": image overlaps an input");
    cudaError_t e = launch_pca_image(C, N, x, mean, components, range, image, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
    return 0;
}
}  // namespace

extern "C" {

int f3dgs_decoder_forward(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x, float* y,
                          void* cuda_stream) {
    return decoder_forward_impl("decoder_forward", Cin, Cout, N, weight, bias, x, y, cuda_stream);
}

int f3dgs_decoder_forward_f16(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                              uint16_t* y, void* cuda_stream) {
    return decoder_forward_impl("decoder_forward_f16", Cin, Cout, N, weight, bias, x, reinterpret_cast<__half*>(y),
                                cuda_stream);
}

int f3dgs_decoder_l1(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x, const float* gt,
                     float grad_scale, float* loss_sum, float* dL_dx, float* dL_dweight, float* dL_dbias,
                     void* cuda_stream) {
    return decoder_l1_impl("decoder_l1", Cin, Cout, N, weight, bias, x, gt, grad_scale, loss_sum, dL_dx, dL_dweight,
                           dL_dbias, cuda_stream);
}

int f3dgs_decoder_l1_f16gt(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                           const uint16_t* gt, float grad_scale, float* loss_sum, float* dL_dx, float* dL_dweight,
                           float* dL_dbias, void* cuda_stream) {
    return decoder_l1_impl("decoder_l1_f16gt", Cin, Cout, N, weight, bias, x, reinterpret_cast<const __half*>(gt),
                           grad_scale, loss_sum, dL_dx, dL_dweight, dL_dbias, cuda_stream);
}

int f3dgs_feature_query(int C, int D, int K, int N, const float* weight, const float* bias, const float* x,
                        const float* text, float logit_scale, const uint8_t* positive, int64_t* labels, float* prob,
                        float* logits, void* cuda_stream) {
    return feature_query_impl("feature_query", C, D, K, N, weight, bias, x, text, logit_scale, positive, labels, prob,
                              logits, cuda_stream);
}

int f3dgs_feature_query_f16x(int C, int D, int K, int N, const float* weight, const float* bias, const uint16_t* x,
                             const float* text, float logit_scale, const uint8_t* positive, int64_t* labels,
                             float* prob, float* logits, void* cuda_stream) {
    return feature_query_impl("feature_query_f16x", C, D, K, N, weight, bias, reinterpret_cast<const __half*>(x), text,
                              logit_scale, positive, labels, prob, logits, cuda_stream);
}

size_t f3dgs_feature_pca_scratch_bytes(int C, int N) {
    t_error.clear();
    if (!pca_sizes_ok(C, N)) return 0;
    size_t bytes = 0;
    const cudaError_t e = pca_scratch_bytes(C, N, &bytes);
    if (e != cudaSuccess) {
        fail(F3DGS_ERR_CUDA, std::string("f3dgs_feature_pca_scratch_bytes: ") + cudaGetErrorString(e));
        return 0;
    }
    return bytes;
}

int f3dgs_feature_pca_moments(int C, int N, const float* x, char* scratch, float* mean, double* cov, void* cuda_stream) {
    return pca_moments_impl("feature_pca_moments", C, N, x, scratch, mean, cov, cuda_stream);
}

int f3dgs_feature_pca_moments_f16x(int C, int N, const uint16_t* x, char* scratch, float* mean, double* cov,
                                   void* cuda_stream) {
    return pca_moments_impl("feature_pca_moments_f16x", C, N, reinterpret_cast<const __half*>(x), scratch, mean, cov,
                            cuda_stream);
}

int f3dgs_feature_pca_range(int C, int N, const float* x, const float* mean, const float* components, char* scratch,
                            float* range, void* cuda_stream) {
    return pca_range_impl("feature_pca_range", C, N, x, mean, components, scratch, range, cuda_stream);
}

int f3dgs_feature_pca_range_f16x(int C, int N, const uint16_t* x, const float* mean, const float* components,
                                 char* scratch, float* range, void* cuda_stream) {
    return pca_range_impl("feature_pca_range_f16x", C, N, reinterpret_cast<const __half*>(x), mean, components, scratch,
                          range, cuda_stream);
}

int f3dgs_feature_pca_image(int C, int N, const float* x, const float* mean, const float* components,
                            const float* range, float* image, void* cuda_stream) {
    return pca_image_impl("feature_pca_image", C, N, x, mean, components, range, image, cuda_stream);
}

int f3dgs_feature_pca_image_f16x(int C, int N, const uint16_t* x, const float* mean, const float* components,
                                 const float* range, float* image, void* cuda_stream) {
    return pca_image_impl("feature_pca_image_f16x", C, N, reinterpret_cast<const __half*>(x), mean, components, range,
                          image, cuda_stream);
}

size_t f3dgs_knn_scratch_bytes(int P) {
    t_error.clear();
    size_t bytes = 0;
    const cudaError_t e = knn_scratch_bytes(P, &bytes);
    if (e != cudaSuccess) {
        fail(F3DGS_ERR_CUDA, std::string("f3dgs_knn_scratch_bytes: ") + cudaGetErrorString(e));
        return 0;
    }
    return bytes;
}

int f3dgs_knn_mean_dist(int P, const float* points, float* out, char* scratch, void* cuda_stream) {
    t_error.clear();
    if (P < 0) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_knn_mean_dist: P < 0");
    if (P == 0) return 0;
    if (!points || !out || !scratch) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_knn_mean_dist: NULL pointer");
    const size_t no = (size_t)P * 4;
    if (ranges_overlap(out, no, points, (size_t)P * 12) || ranges_overlap(out, no, scratch, knn_scratch_fixed_bytes(P)))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_knn_mean_dist: out overlaps points or scratch");
    size_t sb = 0;
    CUDA_TRY(knn_scratch_bytes(P, &sb));  // the sort's share of the scratch is sized by CUB for the current device
    if (ranges_overlap(out, no, scratch, sb))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_knn_mean_dist: out overlaps points or scratch");
    cudaError_t e = launch_knn_mean_dist(P, points, out, scratch, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("knn_mean_dist: ") + cudaGetErrorString(e));
    return 0;
}

size_t f3dgs_densify_scratch_bytes(int P) {
    t_error.clear();
    size_t bytes = 0;
    const cudaError_t e = densify_scratch_bytes(P, &bytes);
    if (e != cudaSuccess) {
        fail(F3DGS_ERR_CUDA, std::string("f3dgs_densify_scratch_bytes: ") + cudaGetErrorString(e));
        return 0;
    }
    return bytes;
}

int f3dgs_densify_plan(int P, const float* grad_accum, const float* denom, const float* raw_opacity,
                       const float* raw_scaling, float max_grad, float dense_scale, float min_opacity,
                       float max_world_scale, char* scratch, int32_t* counts, void* cuda_stream) {
    t_error.clear();
    if (P < 0 || 3 * (long long)P > INT_MAX)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_densify_plan: bad sizes (0 <= 3 P <= INT_MAX)");
    if (!counts || (P > 0 && (!grad_accum || !denom || !raw_opacity || !raw_scaling || !scratch)))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_densify_plan: NULL pointer");
    if (ranges_overlap(counts, 16, scratch, densify_scratch_fixed_bytes(P)))
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_densify_plan: counts overlaps scratch");
    cudaError_t e = launch_densify_plan(P, grad_accum, denom, raw_opacity, raw_scaling, max_grad, dense_scale,
                                        min_opacity, max_world_scale, scratch, counts, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("densify_plan: ") + cudaGetErrorString(e));
    return 0;
}

int f3dgs_densify_apply(int P, int M, int C, const char* scratch, const int32_t counts[4], const float* normals,
                        const f3dgs_gaussian_fields src[3], const f3dgs_gaussian_fields dst[3], void* cuda_stream) {
    t_error.clear();
    if (P < 0 || 3 * (long long)P > INT_MAX || M < 1 || C < 0 || C > F3DGS_MAX_FEATURE_DIM)
        return fail(F3DGS_ERR_INVALID_ARGUMENT,
                    "f3dgs_densify_apply: bad sizes (0 <= 3 P <= INT_MAX, M >= 1, 0 <= C <= F3DGS_MAX_FEATURE_DIM)");
    if (!counts || !src || !dst) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_densify_apply: NULL pointer");
    const long long A = counts[0], B = counts[1], Cc = counts[2], Ns = counts[3], Pn = A + B + 2 * Cc;
    if (A < 0 || B < 0 || Cc < 0 || A > P || B > P || Cc > Ns || Ns > P || 3 * Pn > INT_MAX)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_densify_apply: counts are not those of a plan over P Gaussians");
    if (Ns > 0 && !normals) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_densify_apply: NULL pointer (normals)");
    if (P > 0 && !scratch) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_densify_apply: NULL pointer (scratch)");
    const size_t width[7] = {3, 3, 3 * (size_t)(M - 1), 1, 3, 4, (size_t)C};
    const float* s[21];
    float* d[21];
    for (int g = 0; g < 3; g++) {
        const f3dgs_gaussian_fields* f[2] = {&src[g], &dst[g]};
        for (int k = 0; k < 2; k++) {
            const float* p[7] = {f[k]->xyz, f[k]->f_dc, f[k]->f_rest, f[k]->opacity, f[k]->scaling, f[k]->rotation,
                                 f[k]->semantic_feature};
            for (int j = 0; j < 7; j++) {
                if (width[j] && (k ? Pn : P) > 0 && !p[j])
                    return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_densify_apply: NULL pointer (a src or dst field)");
                if (k) d[7 * g + j] = const_cast<float*>(p[j]);
                else s[7 * g + j] = p[j];
            }
        }
    }
    for (int i = 0; i < 21; i++) {
        const size_t nd = (size_t)Pn * width[i % 7] * 4;
        bool bad = ranges_overlap(d[i], nd, scratch, densify_scratch_fixed_bytes(P)) ||
                   ranges_overlap(d[i], nd, normals, (size_t)Ns * 24);
        for (int j = 0; j < 21 && !bad; j++) bad = ranges_overlap(d[i], nd, s[j], (size_t)P * width[j % 7] * 4);
        if (bad)
            return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_densify_apply: a dst field overlaps a src field, normals or scratch");
    }
    cudaError_t e = launch_densify_apply(P, M, C, scratch, counts, normals, s, d, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("densify_apply: ") + cudaGetErrorString(e));
    return 0;
}

int f3dgs_reset_opacity(int P, float* raw_opacity, float* exp_avg, float* exp_avg_sq, float ceiling, void* cuda_stream) {
    t_error.clear();
    if (P < 0) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_reset_opacity: P < 0");
    if (P == 0) return 0;
    if (!raw_opacity || !exp_avg || !exp_avg_sq) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_reset_opacity: NULL pointer");
    cudaError_t e = launch_reset_opacity(P, raw_opacity, exp_avg, exp_avg_sq, ceiling, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("reset_opacity: ") + cudaGetErrorString(e));
    return 0;
}

int f3dgs_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                       uint8_t* present, void* cuda_stream) {
    (void)projmatrix;  // the reference's frustum side test is commented out (auxiliary.h:160)
    t_error.clear();
    if (P < 0) return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_mark_visible: P < 0");
    if (P == 0) return 0;
    if (!means3D || !viewmatrix || !present)
        return fail(F3DGS_ERR_INVALID_ARGUMENT, "f3dgs_mark_visible: NULL pointer");
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    launch_mark_visible(P, means3D, viewmatrix, present, stream);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(F3DGS_ERR_CUDA, std::string("mark_visible: ") + cudaGetErrorString(e));
    return 0;
}

}  // extern "C"
