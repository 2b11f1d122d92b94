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

// Every entry point that can fail opens an Api named after itself (__func__).  Opening it clears the calling thread's last
// error; a failure records "f3dgs_<entry>: <message>" as the last error and returns the negated error code.
struct Api {
    const char* entry;
    explicit Api(const char* name) : entry(name) { t_error.clear(); }
    int fail(int code, const std::string& msg) const {
        t_error = std::string(entry) + ": " + msg;
        return -code;
    }
    int invalid(const std::string& msg) const { return fail(F3DGS_ERR_INVALID_ARGUMENT, msg); }
    // 0 if a CUDA call or launch succeeded, else its failure, with `what` (if any) naming the step
    int cuda(cudaError_t e, const char* what = nullptr) const {
        if (e == cudaSuccess) return 0;
        return fail(F3DGS_ERR_CUDA, what ? std::string(what) + ": " + cudaGetErrorString(e) : cudaGetErrorString(e));
    }
};

// A byte range [p, p + bytes) of a caller's buffer; a NULL buffer is absent and overlaps nothing.
struct Range {
    const void* p;
    size_t bytes;
};

// Does the output range `out` share a byte with any of the ranges `in`?
template <size_t N>
bool overlaps(const Range& out, const Range (&in)[N]) {
    for (const Range& r : in) {
        const uintptr_t x = (uintptr_t)out.p, y = (uintptr_t)r.p;
        if (out.p && r.p && x < y + r.bytes && y < x + out.bytes) return true;
    }
    return false;
}

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

// The buffers of a forward of the view (R instances) that the composite backward reads
ForwardBuffers forward_buffers(const ViewParams& vp, int R, const char* geom, const char* bin, char* img) {
    const ImgLayout il((size_t)vp.W * vp.H, (size_t)vp.grid_x * vp.grid_y);
    return {reinterpret_cast<const uint2*>(img + il.ranges),
            reinterpret_cast<const uint32_t*>(bin + BinLayout((size_t)R).point_list),
            reinterpret_cast<const SplatRec*>(geom + GeomLayout((size_t)vp.P).rec),
            reinterpret_cast<const float*>(img + il.final_T),
            reinterpret_cast<const uint32_t*>(img + il.n_contrib),
            reinterpret_cast<int*>(img + il.counters),
            R};
}

// Result of a composite-backward call.  It takes its instance lists from the device's default memory pool, so running
// out of memory there is an allocation failure.
int composite_bwd_result(const Api& api, cudaError_t e, const char* what) {
    if (e == cudaErrorMemoryAllocation)
        return api.fail(F3DGS_ERR_ALLOC, std::string("cudaMallocAsync for the instance lists failed: ") +
                                             cudaGetErrorString(e));
    return api.cuda(e, what);
}

inline int bit_length(uint32_t n) {
    int b = 0;
    while (n) {
        b++;
        n >>= 1;
    }
    return b;
}

// both macros report through the entry point's `api`
#define CUDA_TRY(expr)                                                                              \
    do {                                                                                            \
        if (const int rc_ = api.cuda((expr), #expr)) return rc_;                                    \
    } while (0)

// reference CHECK_CUDA (auxiliary.h:172-179): in debug mode synchronise and surface errors per stage
#define STAGE_CHECK(name)                                                                           \
    do {                                                                                            \
        cudaError_t e_ = cudaGetLastError();                                                        \
        if (e_ == cudaSuccess && debug) e_ = cudaStreamSynchronize(stream);                         \
        if (const int rc_ = api.cuda(e_, "stage " name)) return rc_;                                \
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
    const Api api(__func__);
    if (!ms || !count) return api.invalid("NULL output");
    std::lock_guard<std::mutex> lk(g_profile_mu);
    for (const StageRec& r : g_recs) {
        float t = 0.f;
        cudaError_t e = cudaEventSynchronize(r.e1);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&t, r.e0, r.e1);
        if (const int rc = api.cuda(e)) return rc;
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
    const Api api(__func__);
    if (!out || P < 0 || width <= 0 || height <= 0 || R < 0) return api.invalid("bad argument");
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

}  // extern "C"

namespace {

// Shared body of f3dgs_forward (TF = float), f3dgs_forward_f16 (TF = __half), f3dgs_forward_antialiased and
// f3dgs_forward_alpha_invdepth: TF is the element type of semantic_feature and out_feature_map only.  antialiasing:
// op_eff = opacity * rho in the records.  out_alpha / out_invdepth (f3dgs_forward_alpha_invdepth, which has checked that
// both are given): the composite also writes the opacity and inverse-depth planes.
template <typename TF>
int forward_impl(const char* entry, f3dgs_alloc_fn geometry_alloc, void* geometry_ctx, f3dgs_alloc_fn binning_alloc,
                 void* binning_ctx, f3dgs_alloc_fn image_alloc, void* image_ctx, int P, int D, int M, int C,
                 const float* background, int width, int height, const float* means3D, const float* shs,
                 const float* colors_precomp, const TF* semantic_feature, const float* opacities, const float* scales,
                 float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                 const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered,
                 float* out_color, TF* out_feature_map, float* out_depth, int* radii, int debug, void* cuda_stream,
                 bool antialiasing = false, float* out_alpha = nullptr, float* out_invdepth = nullptr) {
    const Api api(entry);
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (P < 0 || width <= 0 || height <= 0 || C < 0 || C > F3DGS_MAX_FEATURE_DIM || D < 0 || D > 3)
        return api.invalid("bad sizes (P, width, height, C or D)");
    if (!geometry_alloc || !binning_alloc || !image_alloc)
        return api.invalid("missing allocator");
    if (P == 0) return 0;
    if (!means3D || !opacities || !background || !viewmatrix || !projmatrix || !cam_pos || !out_color ||
        !out_depth)
        return api.invalid("NULL required pointer");
    if ((shs == nullptr) == (colors_precomp == nullptr))
        return api.invalid("provide exactly one of shs / colors_precomp");
    if (((scales == nullptr) || (rotations == nullptr)) == (cov3D_precomp == nullptr))
        return api.invalid("provide exactly one of (scales, rotations) / cov3D_precomp");
    if (C > 0 && (!semantic_feature || !out_feature_map))
        return api.invalid("C > 0 needs semantic_feature and out_feature_map");
    if (shs && M < (D + 1) * (D + 1)) return api.invalid("M < (D+1)^2 SH coefficients");
    if (out_alpha) {  // the composite writes the planes while it writes the other outputs
        const size_t hw4 = (size_t)width * height * 4;
        const Range a{out_alpha, hw4}, i{out_invdepth, hw4};
        const Range outs[] = {{out_color, 3 * hw4}, {out_feature_map, (size_t)C * width * height * sizeof(TF)},
                              {out_depth, hw4}, {radii, (size_t)P * 4}};
        if (overlaps(a, outs) || overlaps(i, outs) || overlaps(a, {i}))
            return api.invalid("out_alpha / out_invdepth overlap another output");
    }

    const ViewParams vp = make_view(P, D, M, C, width, height, tan_fovx, tan_fovy, scale_modifier, viewmatrix,
                                    projmatrix, cam_pos);
    const size_t tiles = (size_t)vp.grid_x * vp.grid_y;

    // ---- geometry buffer
    const GeomLayout gl((size_t)P);
    size_t scan_bytes = 0;
    CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, P, stream));
    char* geom = geometry_alloc(geometry_ctx, gl.fixed_bytes + align_up(scan_bytes));
    if (!geom) return api.fail(F3DGS_ERR_ALLOC, "geometry allocator returned NULL");
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
    if (!img) return api.fail(F3DGS_ERR_ALLOC, "image allocator returned NULL");
    float* final_T = reinterpret_cast<float*>(img + il.final_T);
    uint32_t* n_contrib = reinterpret_cast<uint32_t*>(img + il.n_contrib);
    uint2* ranges = reinterpret_cast<uint2*>(img + il.ranges);

    {
        StageTimer t(F3DGS_STAGE_PREPROCESS_FWD, stream);
        launch_preprocess_fwd(vp, means3D, scales, rotations, opacities, shs, cov3D_precomp, colors_precomp,
                              prefiltered != 0, radii, rec, cov3d, clamped, tiles_touched, stream, antialiasing);
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
    if (R < 0) return api.fail(F3DGS_ERR_CUDA, "num_rendered overflowed int32");

    // ---- binning buffer
    const BinLayout bl((size_t)R);
    const int end_bit = 32 + bit_length((uint32_t)(tiles > 0 ? tiles - 1 : 0));
    size_t sort_bytes = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr,
                                             (uint32_t*)nullptr, (uint32_t*)nullptr, R, 0, end_bit, stream));
    char* bin = binning_alloc(binning_ctx, bl.fixed_bytes + align_up(sort_bytes));
    if (!bin) return api.fail(F3DGS_ERR_ALLOC, "binning allocator returned NULL");
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
                                 out_color, out_feature_map, out_depth, counters, stream, out_alpha, out_invdepth);
    }
    if (const int rc = api.cuda(e, "composite_fwd launch")) return rc;
    STAGE_CHECK("composite_fwd");
    return R;
}

}  // namespace

extern "C" {

int f3dgs_forward(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx, f3dgs_alloc_fn binning_alloc,
                  void* binning_ctx, f3dgs_alloc_fn image_alloc, void* image_ctx, int P, int D, int M, int C,
                  const float* background, int width, int height, const float* means3D, const float* shs,
                  const float* colors_precomp, const float* semantic_feature, const float* opacities,
                  const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
                  const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                  float tan_fovy, int prefiltered, float* out_color, float* out_feature_map, float* out_depth,
                  int* radii, int debug, void* cuda_stream) {
    return forward_impl(__func__, geometry_alloc, geometry_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx, P,
                        D, M, C, background, width, height, means3D, shs, colors_precomp, semantic_feature, opacities,
                        scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                        tan_fovy, prefiltered, out_color, out_feature_map, out_depth, radii, debug, cuda_stream);
}

int f3dgs_forward_f16(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx, f3dgs_alloc_fn binning_alloc,
                      void* binning_ctx, f3dgs_alloc_fn image_alloc, void* image_ctx, int P, int D, int M, int C,
                      const float* background, int width, int height, const float* means3D, const float* shs,
                      const float* colors_precomp, const uint16_t* semantic_feature, const float* opacities,
                      const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
                      const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                      float tan_fovy, int prefiltered, float* out_color, uint16_t* out_feature_map, float* out_depth,
                      int* radii, int debug, void* cuda_stream) {
    return forward_impl(__func__, geometry_alloc, geometry_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx, P,
                        D, M, C, background, width, height, means3D, shs, colors_precomp,
                        reinterpret_cast<const __half*>(semantic_feature), opacities, scales, scale_modifier, rotations,
                        cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered, out_color,
                        reinterpret_cast<__half*>(out_feature_map), out_depth, radii, debug, cuda_stream);
}

int f3dgs_forward_antialiased(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx, f3dgs_alloc_fn binning_alloc,
                              void* binning_ctx, f3dgs_alloc_fn image_alloc, void* image_ctx, int P, int D, int M,
                              int C, const float* background, int width, int height, const float* means3D,
                              const float* shs, const float* colors_precomp, const void* semantic_feature,
                              int semantic_feature_dtype, const float* opacities, const float* scales,
                              float scale_modifier, const float* rotations, const float* cov3D_precomp,
                              const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                              float tan_fovy, int prefiltered, float* out_color, void* out_feature_map,
                              float* out_depth, int* radii, int debug, void* cuda_stream) {
    const char* entry = __func__;
    const auto run = [&](auto* features) {
        using TF = std::remove_const_t<std::remove_pointer_t<decltype(features)>>;
        return forward_impl(entry, geometry_alloc, geometry_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx,
                            P, D, M, C, background, width, height, means3D, shs, colors_precomp, features, opacities,
                            scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                            tan_fovy, prefiltered, out_color, static_cast<TF*>(out_feature_map), out_depth, radii,
                            debug, cuda_stream, true);
    };
    if (semantic_feature_dtype == F3DGS_F32) return run(static_cast<const float*>(semantic_feature));
    if (semantic_feature_dtype == F3DGS_F16) return run(static_cast<const __half*>(semantic_feature));
    return Api(__func__).invalid("unknown dtype code");
}

int f3dgs_forward_alpha_invdepth(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx, f3dgs_alloc_fn binning_alloc,
                                 void* binning_ctx, f3dgs_alloc_fn image_alloc, void* image_ctx, int P, int D, int M,
                                 int C, const float* background, int width, int height, const float* means3D,
                                 const float* shs, const float* colors_precomp, const void* semantic_feature,
                                 int semantic_feature_dtype, const float* opacities, const float* scales,
                                 float scale_modifier, const float* rotations, const float* cov3D_precomp,
                                 const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                 float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                                 void* out_feature_map, float* out_depth, int* radii, int debug, void* cuda_stream,
                                 int antialiasing, float* out_alpha, float* out_invdepth) {
    const char* entry = __func__;
    if (!out_alpha || !out_invdepth) return Api(entry).invalid("NULL out_alpha / out_invdepth");
    const auto run = [&](auto* features) {
        using TF = std::remove_const_t<std::remove_pointer_t<decltype(features)>>;
        return forward_impl(entry, geometry_alloc, geometry_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx,
                            P, D, M, C, background, width, height, means3D, shs, colors_precomp, features, opacities,
                            scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                            tan_fovy, prefiltered, out_color, static_cast<TF*>(out_feature_map), out_depth, radii,
                            debug, cuda_stream, antialiasing != 0, out_alpha, out_invdepth);
    };
    if (semantic_feature_dtype == F3DGS_F32) return run(static_cast<const float*>(semantic_feature));
    if (semantic_feature_dtype == F3DGS_F16) return run(static_cast<const __half*>(semantic_feature));
    return Api(entry).invalid("unknown dtype code");
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

// Shared body of f3dgs_backward (accumulate = false: the reference's assign-into-zeroed-buffers contract),
// f3dgs_backward_accum (accumulate = true: += into the caller's per-parameter gradient buffers) and their _f16 twins.
// TG (float or __half) is the element type of dL_dfeaturepix; a __half map stands for dL/dO = scale * float(h).
// `zero` (accumulate only): the caller's scratch, zeroed once the arguments are validated.  feat.rows (the _feature_geometry
// entries only; NULL on every other path): the Gaussians' features, for the feature term of dL/dalpha.  antialiasing
// (the _antialiased entries): the forward's records hold op_eff = opacity * rho, so the composite's opacity gradient is
// dL/dop_eff and the preprocess backward turns it into dL/dopacity (and rho's geometric terms).  The assigning backward
// lets the composite write into dL_dopacity and rescales it in place; the accumulating one needs dL/dop_eff of this view
// alone, so the composite writes into P zeroed floats of the device's default memory pool.  dL_dalpha / dL_dinvdepth
// (the _alpha_invdepth entries, which have checked that both are given): the gradients of the forward's opacity and
// inverse-depth planes, added to dL/dalpha and dL/dz by the composite.
template <typename TG>
int backward_impl(const Api& api, bool accumulate, int P, int D, int M, int R, int C, const float* background, int width,
                  int height, const float* means3D, const float* shs, const float* scales, float scale_modifier,
                  const float* rotations, const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                  const float* cam_pos, float tan_fovx, float tan_fovy, const int* radii, char* geom_buffer,
                  char* binning_buffer, char* image_buffer, const float* dL_dpix, const TG* dL_dfeaturepix,
                  float dL_dfeaturepix_scale, const float* dL_depths, float* dL_dmean2D, float* dL_dconic,
                  float* dL_dopacity, float* dL_dcolor, float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                  float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz, float* grad_accum, float* denom,
                  float* dL_dcamera, cudaEvent_t composite_done, int debug, cudaStream_t stream,
                  const Range& zero = {nullptr, 0}, const FeatureRows& feat = {}, bool antialiasing = false,
                  const float* dL_dalpha = nullptr, const float* dL_dinvdepth = nullptr) {
    if (P < 0 || width <= 0 || height <= 0 || C < 0 || C > F3DGS_MAX_FEATURE_DIM || R < 0)
        return api.invalid("bad sizes");
    if (P == 0) return 0;
    if (!geom_buffer || !binning_buffer || !image_buffer) return api.invalid("missing forward buffers");
    if (!dL_dpix || !dL_depths || (C > 0 && (!dL_dfeaturepix || !dL_dsemantic_feature)) || !dL_dmean2D ||
        !dL_dconic || !dL_dopacity || !dL_dcolor || !dL_dmean3D || !dL_dcov3D || !dL_dz)
        return api.invalid("NULL gradient pointer");
    if (shs && !dL_dsh) return api.invalid("shs given but dL_dsh NULL");
    if (scales && (!rotations || !dL_dscale || !dL_drot))
        return api.invalid("scales given but rotations/dL_dscale/dL_drot NULL");
    if ((grad_accum == nullptr) != (denom == nullptr)) return api.invalid("grad_accum and denom go together");
    if constexpr (std::is_same_v<TG, __half>) {
        if (!std::isfinite(dL_dfeaturepix_scale) || dL_dfeaturepix_scale == 0.f)
            return api.invalid("dL_dfeaturepix_scale must be finite and nonzero");
        // the feature kernel reduces into dL_dsemantic_feature while other warps still read the map
        if (overlaps({dL_dsemantic_feature, (size_t)P * C * 4}, {{dL_dfeaturepix, (size_t)C * width * height * 2}}))
            return api.invalid("dL_dsemantic_feature overlaps dL_dfeaturepix");
    }
    if (dL_dcamera) {
        const size_t p4 = (size_t)P * 4;
        const Range outs[] = {{dL_dmean2D, 3 * p4}, {dL_dconic, 4 * p4}, {dL_dopacity, p4}, {dL_dcolor, 3 * p4},
                              {dL_dsemantic_feature, (size_t)C * p4}, {dL_dmean3D, 3 * p4}, {dL_dcov3D, 6 * p4},
                              {dL_dsh, (size_t)M * 3 * p4}, {dL_dscale, 3 * p4}, {dL_drot, 4 * p4}, {dL_dz, p4},
                              {grad_accum, p4}, {denom, p4}, zero};
        if (overlaps({dL_dcamera, F3DGS_CAMERA_GRAD_FLOATS * sizeof(float)}, outs))
            return api.invalid("dL_dcamera overlaps another output");
    }
    if (feat.rows) {
        const size_t p4 = (size_t)P * 4;
        const Range outs[] = {{dL_dmean2D, 3 * p4}, {dL_dconic, 4 * p4}, {dL_dopacity, p4}, {dL_dcolor, 3 * p4},
                              {dL_dsemantic_feature, (size_t)C * p4}, {dL_dmean3D, 3 * p4}, {dL_dcov3D, 6 * p4},
                              {dL_dsh, (size_t)M * 3 * p4}, {dL_dscale, 3 * p4}, {dL_drot, 4 * p4}, {dL_dz, p4},
                              {grad_accum, p4}, {denom, p4}, {dL_dcamera, F3DGS_CAMERA_GRAD_FLOATS * sizeof(float)},
                              zero};
        if (overlaps({feat.rows, (size_t)P * C * (feat.f16 ? 2 : 4)}, outs))
            return api.invalid("semantic_feature overlaps an output");
    }
    if (antialiasing) {  // the preprocess backward writes dL_dopacity while it writes the others
        const size_t p4 = (size_t)P * 4;
        const Range outs[] = {{dL_dmean2D, 3 * p4}, {dL_dconic, 4 * p4}, {dL_dcolor, 3 * p4},
                              {dL_dsemantic_feature, (size_t)C * p4}, {dL_dmean3D, 3 * p4}, {dL_dcov3D, 6 * p4},
                              {dL_dsh, (size_t)M * 3 * p4}, {dL_dscale, 3 * p4}, {dL_drot, 4 * p4}, {dL_dz, p4},
                              {grad_accum, p4}, {denom, p4}, {dL_dcamera, F3DGS_CAMERA_GRAD_FLOATS * sizeof(float)},
                              zero};
        if (overlaps({dL_dopacity, p4}, outs)) return api.invalid("dL_dopacity overlaps another output");
    }
    if (dL_dalpha) {  // read by the composite while it reduces into the outputs
        const size_t p4 = (size_t)P * 4, hw4 = (size_t)width * height * 4;
        const Range outs[] = {{dL_dmean2D, 3 * p4}, {dL_dconic, 4 * p4}, {dL_dopacity, p4}, {dL_dcolor, 3 * p4},
                              {dL_dsemantic_feature, (size_t)C * p4}, {dL_dmean3D, 3 * p4}, {dL_dcov3D, 6 * p4},
                              {dL_dsh, (size_t)M * 3 * p4}, {dL_dscale, 3 * p4}, {dL_drot, 4 * p4}, {dL_dz, p4},
                              {grad_accum, p4}, {denom, p4}, {dL_dcamera, F3DGS_CAMERA_GRAD_FLOATS * sizeof(float)},
                              zero};
        if (overlaps({dL_dalpha, hw4}, outs) || overlaps({dL_dinvdepth, hw4}, outs))
            return api.invalid("dL_dalpha / dL_dinvdepth overlap an output");
    }
    if (zero.p) CUDA_TRY(cudaMemsetAsync(const_cast<void*>(zero.p), 0, zero.bytes, stream));

    const ViewParams vp = make_view(P, D, M, C, width, height, tan_fovx, tan_fovy, scale_modifier, viewmatrix,
                                    projmatrix, cam_pos);
    const GeomLayout gl((size_t)P);
    const float* cov3d = cov3D_precomp ? cov3D_precomp : reinterpret_cast<const float*>(geom_buffer + gl.cov3d);
    const uint8_t* clamped = reinterpret_cast<const uint8_t*>(geom_buffer + gl.clamped);
    if (radii == nullptr) radii = reinterpret_cast<const int*>(geom_buffer + gl.radii);

    cudaError_t e;
    // where the composite puts the opacity gradient: dL/dop_eff under antialiasing (see above)
    struct PoolFloats {  // returned to the pool on every exit
        float* p = nullptr;
        cudaStream_t s;
        ~PoolFloats() {
            if (p) cudaFreeAsync(p, s);
        }
    } op_eff_grad{nullptr, stream};
    float* dL_dop_eff = dL_dopacity;
    if (antialiasing && accumulate) {
        e = cudaMallocAsync((void**)&op_eff_grad.p, (size_t)P * sizeof(float), stream);
        if (e != cudaSuccess)
            return api.fail(F3DGS_ERR_ALLOC, std::string("cudaMallocAsync for dL/dop_eff failed: ") +
                                                 cudaGetErrorString(e));
        CUDA_TRY(cudaMemsetAsync(op_eff_grad.p, 0, (size_t)P * sizeof(float), stream));
        dL_dop_eff = op_eff_grad.p;
    }
    {
        StageTimer t(F3DGS_STAGE_COMPOSITE_BWD, stream);
        e = launch_composite_bwd(vp, forward_buffers(vp, R, geom_buffer, binning_buffer, image_buffer), background,
                                 dL_dpix, dL_depths, dL_dfeaturepix, dL_dfeaturepix_scale, dL_dmean2D, dL_dconic,
                                 dL_dop_eff, dL_dcolor, dL_dz, dL_dsemantic_feature, stream, feat, dL_dalpha,
                                 dL_dinvdepth);
    }
    if (const int rc = composite_bwd_result(api, e, "composite_bwd launch")) return rc;
    STAGE_CHECK("composite_bwd");
    // dL_dopacity is final after the composite, or under antialiasing after the preprocess backward
    if (composite_done && !antialiasing) CUDA_TRY(cudaEventRecord(composite_done, stream));
    {
        StageTimer t(F3DGS_STAGE_PREPROCESS_BWD, stream);
        e = launch_preprocess_bwd(vp, means3D, radii, shs, clamped, scales, rotations, cov3d, dL_dmean2D, dL_dconic,
                                  dL_dmean3D, dL_dcolor, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dz, stream,
                                  accumulate, grad_accum, denom, dL_dcamera, antialiasing,
                                  reinterpret_cast<const SplatRec*>(geom_buffer + gl.rec), dL_dop_eff, dL_dopacity);
    }
    if (e == cudaErrorMemoryAllocation)
        return api.fail(F3DGS_ERR_ALLOC, std::string("cudaMallocAsync for the camera-gradient partials failed: ") +
                                             cudaGetErrorString(e));
    CUDA_TRY(e);
    STAGE_CHECK("preprocess_bwd");
    if (composite_done && antialiasing) CUDA_TRY(cudaEventRecord(composite_done, stream));
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
    return backward_impl(Api(__func__), false, P, D, M, R, C, background, width, height, means3D, shs, scales,
                         scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy,
                         radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, dL_dfeaturepix, 1.f, dL_depths,
                         dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh,
                         dL_dscale, dL_drot, dL_dz, nullptr, nullptr, nullptr, nullptr, debug, (cudaStream_t)cuda_stream);
}

int f3dgs_backward_f16(int P, int D, int M, int R, int C, const float* background, int width, int height,
                       const float* means3D, const float* shs, const float* colors_precomp,
                       const float* semantic_feature, const float* scales, float scale_modifier,
                       const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                       const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
                       const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                       const float* dL_dpix, const uint16_t* dL_dfeaturepix, float dL_dfeaturepix_scale,
                       const float* dL_depths, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                       float* dL_dcolor, float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                       float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz, int debug, void* cuda_stream) {
    (void)semantic_feature;
    (void)colors_precomp;
    return backward_impl(Api(__func__), false, P, D, M, R, C, background, width, height, means3D, shs, scales,
                         scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy,
                         radii, geom_buffer, binning_buffer, image_buffer, dL_dpix,
                         reinterpret_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale, dL_depths, dL_dmean2D,
                         dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
                         dL_drot, dL_dz, nullptr, nullptr, nullptr, nullptr, debug, (cudaStream_t)cuda_stream);
}

int f3dgs_backward_cam(int P, int D, int M, int R, int C, const float* background, int width, int height,
                       const float* means3D, const float* shs, const float* colors_precomp,
                       const float* semantic_feature, const float* scales, float scale_modifier,
                       const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                       const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
                       const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                       const float* dL_dpix, const float* dL_dfeaturepix, const float* dL_depths, float* dL_dmean2D,
                       float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dsemantic_feature,
                       float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                       float* dL_dz, int debug, void* cuda_stream, float* dL_dcamera) {
    (void)semantic_feature;
    (void)colors_precomp;
    const Api api(__func__);
    if (!dL_dcamera) return api.invalid("NULL dL_dcamera");
    return backward_impl(api, false, P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier,
                         rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii,
                         geom_buffer, binning_buffer, image_buffer, dL_dpix, dL_dfeaturepix, 1.f, dL_depths, dL_dmean2D,
                         dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh,
                         dL_dscale, dL_drot, dL_dz, nullptr, nullptr, dL_dcamera, nullptr, debug,
                         (cudaStream_t)cuda_stream);
}

int f3dgs_backward_cam_f16(int P, int D, int M, int R, int C, const float* background, int width, int height,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* semantic_feature, const float* scales, float scale_modifier,
                           const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                           const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
                           const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                           const float* dL_dpix, const uint16_t* dL_dfeaturepix, float dL_dfeaturepix_scale,
                           const float* dL_depths, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                           float* dL_dcolor, float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                           float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz, int debug,
                           void* cuda_stream, float* dL_dcamera) {
    (void)semantic_feature;
    (void)colors_precomp;
    const Api api(__func__);
    if (!dL_dcamera) return api.invalid("NULL dL_dcamera");
    return backward_impl(api, false, P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier,
                         rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii,
                         geom_buffer, binning_buffer, image_buffer, dL_dpix,
                         reinterpret_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale, dL_depths, dL_dmean2D,
                         dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh,
                         dL_dscale, dL_drot, dL_dz, nullptr, nullptr, dL_dcamera, nullptr, debug,
                         (cudaStream_t)cuda_stream);
}

size_t f3dgs_backward_scratch_bytes(int P) { return P > 0 ? ScratchLayout((size_t)P).bytes : 0; }

}  // extern "C"

namespace {
// Shared body of f3dgs_backward_accum and f3dgs_backward_accum_f16 (TG as in backward_impl)
template <typename TG>
int backward_accum_impl(const char* entry, int P, int D, int M, int R, int C, const float* background, int width,
                        int height, const float* means3D, const float* shs, const float* colors_precomp,
                        const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
                        const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                        float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                        const float* dL_dpix, const TG* dL_dfeaturepix, float dL_dfeaturepix_scale,
                        const float* dL_depths, char* scratch, float* dL_dopacity, float* dL_dcolors_precomp,
                        float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh,
                        float* dL_dscale, float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                        void* composite_done_event, int debug, void* cuda_stream, bool camera = false,
                        float* dL_dcamera = nullptr, const FeatureRows& feat = {}, bool antialiasing = false,
                        const float* dL_dalpha = nullptr, const float* dL_dinvdepth = nullptr) {
    const Api api(entry);
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (camera && !dL_dcamera) return api.invalid("NULL dL_dcamera");
    if (P <= 0) return P == 0 ? 0 : api.invalid("bad sizes");
    if (!scratch) return api.invalid("NULL scratch");
    if (overlaps({dL_dcamera, F3DGS_CAMERA_GRAD_FLOATS * sizeof(float)}, {{dL_dmean2D_out, (size_t)P * 3 * 4}}))
        return api.invalid("dL_dcamera overlaps another output");
    if (overlaps({feat.rows, (size_t)P * C * (feat.f16 ? 2 : 4)}, {{dL_dmean2D_out, (size_t)P * 3 * 4}}))
        return api.invalid("semantic_feature overlaps an output");
    const size_t hw4 = (size_t)width * height * 4;
    if (overlaps({dL_dalpha, hw4}, {{dL_dmean2D_out, (size_t)P * 3 * 4}}) ||
        overlaps({dL_dinvdepth, hw4}, {{dL_dmean2D_out, (size_t)P * 3 * 4}}))
        return api.invalid("dL_dalpha / dL_dinvdepth overlap an output");
    if ((colors_precomp != nullptr) != (dL_dcolors_precomp != nullptr) ||
        (cov3D_precomp != nullptr) != (dL_dcov3D_precomp != nullptr))
        return api.invalid("dL_dcolors_precomp / dL_dcov3D_precomp go with colors_precomp / cov3D_precomp");
    const ScratchLayout sl((size_t)P);
    float* m2d = reinterpret_cast<float*>(scratch + sl.mean2D);
    // colours / cov3D are intermediates unless they are inputs of the caller (then their gradients accumulate)
    float* dcol = dL_dcolors_precomp ? dL_dcolors_precomp : reinterpret_cast<float*>(scratch + sl.color);
    float* dcov = dL_dcov3D_precomp ? dL_dcov3D_precomp : reinterpret_cast<float*>(scratch + sl.cov3D);
    const int rc = backward_impl(
        api, true, P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier,
        rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
        binning_buffer, image_buffer, dL_dpix, dL_dfeaturepix, dL_dfeaturepix_scale, dL_depths, m2d,
        reinterpret_cast<float*>(scratch + sl.conic), dL_dopacity, dcol, dL_dsemantic_feature, dL_dmean3D, dcov, dL_dsh,
        dL_dscale, dL_drot, reinterpret_cast<float*>(scratch + sl.dz), grad_accum, denom, dL_dcamera,
        (cudaEvent_t)composite_done_event, debug, stream, {scratch, sl.bytes}, feat, antialiasing, dL_dalpha,
        dL_dinvdepth);
    if (rc < 0) return rc;
    if (dL_dmean2D_out)
        CUDA_TRY(cudaMemcpyAsync(dL_dmean2D_out, m2d, (size_t)P * 3 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    return 0;
}
}  // namespace

extern "C" {

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
    return backward_accum_impl(__func__, P, D, M, R, C, background, width, height, means3D, shs, colors_precomp, scales,
                               scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                               tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, dL_dfeaturepix, 1.f,
                               dL_depths, scratch, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D,
                               dL_dcov3D_precomp, dL_dsh, dL_dscale, dL_drot, dL_dmean2D_out, grad_accum, denom,
                               composite_done_event, debug, cuda_stream);
}

int f3dgs_backward_accum_f16(int P, int D, int M, int R, int C, const float* background, int width, int height,
                             const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                             float scale_modifier, const float* rotations, const float* cov3D_precomp,
                             const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                             float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer,
                             char* image_buffer, const float* dL_dpix, const uint16_t* dL_dfeaturepix,
                             float dL_dfeaturepix_scale, const float* dL_depths, char* scratch, float* dL_dopacity,
                             float* dL_dcolors_precomp, float* dL_dsemantic_feature, float* dL_dmean3D,
                             float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale, float* dL_drot,
                             float* dL_dmean2D_out, float* grad_accum, float* denom, void* composite_done_event,
                             int debug, void* cuda_stream) {
    return backward_accum_impl(__func__, P, D, M, R, C, background, width, height, means3D, shs, colors_precomp, scales,
                               scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                               tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix,
                               reinterpret_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale, dL_depths, scratch,
                               dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D_precomp,
                               dL_dsh, dL_dscale, dL_drot, dL_dmean2D_out, grad_accum, denom, composite_done_event, debug,
                               cuda_stream);
}

int f3dgs_backward_accum_cam(int P, int D, int M, int R, int C, const float* background, int width, int height,
                             const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                             float scale_modifier, const float* rotations, const float* cov3D_precomp,
                             const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                             float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer,
                             char* image_buffer, const float* dL_dpix, const float* dL_dfeaturepix,
                             const float* dL_depths, char* scratch, float* dL_dopacity, float* dL_dcolors_precomp,
                             float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh,
                             float* dL_dscale, float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                             void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera) {
    return backward_accum_impl(__func__, P, D, M, R, C, background, width, height, means3D, shs, colors_precomp, scales,
                               scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                               tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, dL_dfeaturepix, 1.f,
                               dL_depths, scratch, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D,
                               dL_dcov3D_precomp, dL_dsh, dL_dscale, dL_drot, dL_dmean2D_out, grad_accum, denom,
                               composite_done_event, debug, cuda_stream, true, dL_dcamera);
}

int f3dgs_backward_accum_cam_f16(int P, int D, int M, int R, int C, const float* background, int width, int height,
                                 const float* means3D, const float* shs, const float* colors_precomp,
                                 const float* scales, float scale_modifier, const float* rotations,
                                 const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                                 const float* cam_pos, float tan_fovx, float tan_fovy, const int* radii,
                                 char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                                 const uint16_t* dL_dfeaturepix, float dL_dfeaturepix_scale, const float* dL_depths,
                                 char* scratch, float* dL_dopacity, float* dL_dcolors_precomp,
                                 float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D_precomp,
                                 float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dmean2D_out,
                                 float* grad_accum, float* denom, void* composite_done_event, int debug,
                                 void* cuda_stream, float* dL_dcamera) {
    return backward_accum_impl(__func__, P, D, M, R, C, background, width, height, means3D, shs, colors_precomp, scales,
                               scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                               tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix,
                               reinterpret_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale, dL_depths, scratch,
                               dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D_precomp,
                               dL_dsh, dL_dscale, dL_drot, dL_dmean2D_out, grad_accum, denom, composite_done_event, debug,
                               cuda_stream, true, dL_dcamera);
}

}  // extern "C"

namespace {
// The Gaussians' features of a _feature_geometry or _antialiased entry, after the checks every such entry makes before
// any launch.  `optional` (the _antialiased entries): a NULL semantic_feature means no feature term.
int feature_rows(const Api& api, int C, const void* semantic_feature, int semantic_feature_dtype,
                 int dL_dfeaturepix_dtype, FeatureRows& feat, bool optional = false) {
    const auto known = [](int t) { return t == F3DGS_F32 || t == F3DGS_F16; };
    if (!known(semantic_feature_dtype) || !known(dL_dfeaturepix_dtype)) return api.invalid("unknown dtype code");
    if (C > 0 && !semantic_feature && !optional) return api.invalid("NULL semantic_feature");
    feat = {C > 0 ? semantic_feature : nullptr, semantic_feature_dtype == F3DGS_F16};
    return 0;
}
}  // namespace

extern "C" {

int f3dgs_backward_feature_geometry(int P, int D, int M, int R, int C, const float* background, int width, int height,
                                    const float* means3D, const float* shs, const float* colors_precomp,
                                    const void* semantic_feature, int semantic_feature_dtype, const float* scales,
                                    float scale_modifier, const float* rotations, const float* cov3D_precomp,
                                    const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                    float tan_fovx, float tan_fovy, const int* radii, char* geom_buffer,
                                    char* binning_buffer, char* image_buffer, const float* dL_dpix,
                                    const void* dL_dfeaturepix, int dL_dfeaturepix_dtype, float dL_dfeaturepix_scale,
                                    const float* dL_depths, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                                    float* dL_dcolor, float* dL_dsemantic_feature, float* dL_dmean3D,
                                    float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz,
                                    int debug, void* cuda_stream, float* dL_dcamera) {
    (void)colors_precomp;
    const Api api(__func__);
    FeatureRows feat;
    if (const int rc = feature_rows(api, C, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype, feat))
        return rc;
    const auto run = [&](auto map, float scale) {
        return backward_impl(api, false, P, D, M, R, C, background, width, height, means3D, shs, scales,
                             scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                             tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, map, scale, dL_depths,
                             dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D,
                             dL_dsh, dL_dscale, dL_drot, dL_dz, nullptr, nullptr, dL_dcamera, nullptr, debug,
                             (cudaStream_t)cuda_stream, {nullptr, 0}, feat);
    };
    if (dL_dfeaturepix_dtype == F3DGS_F16)
        return run(static_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale);
    return run(static_cast<const float*>(dL_dfeaturepix), 1.f);
}

int f3dgs_backward_accum_feature_geometry(
    int P, int D, int M, int R, int C, const float* background, int width, int height, const float* means3D,
    const float* shs, const float* colors_precomp, const void* semantic_feature, int semantic_feature_dtype,
    const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
    const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
    const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
    const void* dL_dfeaturepix, int dL_dfeaturepix_dtype, float dL_dfeaturepix_scale, const float* dL_depths,
    char* scratch, float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature, float* dL_dmean3D,
    float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dmean2D_out,
    float* grad_accum, float* denom, void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera) {
    const char* entry = __func__;
    FeatureRows feat;
    if (const int rc = feature_rows(Api(entry), C, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype,
                                    feat))
        return rc;
    const auto run = [&](auto map, float scale) {
        return backward_accum_impl(entry, P, D, M, R, C, background, width, height, means3D, shs, colors_precomp,
                                   scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos,
                                   tan_fovx, tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, map,
                                   scale, dL_depths, scratch, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature,
                                   dL_dmean3D, dL_dcov3D_precomp, dL_dsh, dL_dscale, dL_drot, dL_dmean2D_out,
                                   grad_accum, denom, composite_done_event, debug, cuda_stream, false, dL_dcamera,
                                   feat);
    };
    if (dL_dfeaturepix_dtype == F3DGS_F16)
        return run(static_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale);
    return run(static_cast<const float*>(dL_dfeaturepix), 1.f);
}

int f3dgs_backward_antialiased(int P, int D, int M, int R, int C, const float* background, int width, int height,
                               const float* means3D, const float* shs, const float* colors_precomp,
                               const void* semantic_feature, int semantic_feature_dtype, const float* scales,
                               float scale_modifier, const float* rotations, const float* cov3D_precomp,
                               const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                               float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer,
                               char* image_buffer, const float* dL_dpix, const void* dL_dfeaturepix,
                               int dL_dfeaturepix_dtype, float dL_dfeaturepix_scale, const float* dL_depths,
                               float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                               float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                               float* dL_dscale, float* dL_drot, float* dL_dz, int debug, void* cuda_stream,
                               float* dL_dcamera) {
    (void)colors_precomp;
    const Api api(__func__);
    FeatureRows feat;
    if (const int rc =
            feature_rows(api, C, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype, feat, true))
        return rc;
    const auto run = [&](auto map, float scale) {
        return backward_impl(api, false, P, D, M, R, C, background, width, height, means3D, shs, scales,
                             scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                             tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, map, scale, dL_depths,
                             dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D,
                             dL_dsh, dL_dscale, dL_drot, dL_dz, nullptr, nullptr, dL_dcamera, nullptr, debug,
                             (cudaStream_t)cuda_stream, {nullptr, 0}, feat, true);
    };
    if (dL_dfeaturepix_dtype == F3DGS_F16)
        return run(static_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale);
    return run(static_cast<const float*>(dL_dfeaturepix), 1.f);
}

int f3dgs_backward_accum_antialiased(
    int P, int D, int M, int R, int C, const float* background, int width, int height, const float* means3D,
    const float* shs, const float* colors_precomp, const void* semantic_feature, int semantic_feature_dtype,
    const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
    const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
    const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
    const void* dL_dfeaturepix, int dL_dfeaturepix_dtype, float dL_dfeaturepix_scale, const float* dL_depths,
    char* scratch, float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature, float* dL_dmean3D,
    float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dmean2D_out,
    float* grad_accum, float* denom, void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera) {
    const char* entry = __func__;
    FeatureRows feat;
    if (const int rc = feature_rows(Api(entry), C, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype,
                                    feat, true))
        return rc;
    if (P > 0 && overlaps({dL_dopacity, (size_t)P * 4}, {{dL_dmean2D_out, (size_t)P * 3 * 4}}))
        return Api(entry).invalid("dL_dopacity overlaps another output");
    const auto run = [&](auto map, float scale) {
        return backward_accum_impl(entry, P, D, M, R, C, background, width, height, means3D, shs, colors_precomp,
                                   scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos,
                                   tan_fovx, tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, map,
                                   scale, dL_depths, scratch, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature,
                                   dL_dmean3D, dL_dcov3D_precomp, dL_dsh, dL_dscale, dL_drot, dL_dmean2D_out,
                                   grad_accum, denom, composite_done_event, debug, cuda_stream, false, dL_dcamera,
                                   feat, true);
    };
    if (dL_dfeaturepix_dtype == F3DGS_F16)
        return run(static_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale);
    return run(static_cast<const float*>(dL_dfeaturepix), 1.f);
}

int f3dgs_backward_alpha_invdepth(int P, int D, int M, int R, int C, const float* background, int width, int height,
                                  const float* means3D, const float* shs, const float* colors_precomp,
                                  const void* semantic_feature, int semantic_feature_dtype, const float* scales,
                                  float scale_modifier, const float* rotations, const float* cov3D_precomp,
                                  const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                  float tan_fovx, float tan_fovy, const int* radii, char* geom_buffer,
                                  char* binning_buffer, char* image_buffer, const float* dL_dpix,
                                  const void* dL_dfeaturepix, int dL_dfeaturepix_dtype, float dL_dfeaturepix_scale,
                                  const float* dL_depths, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                                  float* dL_dcolor, float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                                  float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz, int debug,
                                  void* cuda_stream, float* dL_dcamera, int antialiasing, const float* dL_dalpha,
                                  const float* dL_dinvdepth) {
    (void)colors_precomp;
    const Api api(__func__);
    if (!dL_dalpha || !dL_dinvdepth) return api.invalid("NULL dL_dalpha / dL_dinvdepth");
    FeatureRows feat;
    if (const int rc =
            feature_rows(api, C, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype, feat, true))
        return rc;
    const auto run = [&](auto map, float scale) {
        return backward_impl(api, false, P, D, M, R, C, background, width, height, means3D, shs, scales,
                             scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                             tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, map, scale, dL_depths,
                             dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D,
                             dL_dsh, dL_dscale, dL_drot, dL_dz, nullptr, nullptr, dL_dcamera, nullptr, debug,
                             (cudaStream_t)cuda_stream, {nullptr, 0}, feat, antialiasing != 0, dL_dalpha,
                             dL_dinvdepth);
    };
    if (dL_dfeaturepix_dtype == F3DGS_F16)
        return run(static_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale);
    return run(static_cast<const float*>(dL_dfeaturepix), 1.f);
}

int f3dgs_backward_accum_alpha_invdepth(
    int P, int D, int M, int R, int C, const float* background, int width, int height, const float* means3D,
    const float* shs, const float* colors_precomp, const void* semantic_feature, int semantic_feature_dtype,
    const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
    const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
    const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
    const void* dL_dfeaturepix, int dL_dfeaturepix_dtype, float dL_dfeaturepix_scale, const float* dL_depths,
    char* scratch, float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature, float* dL_dmean3D,
    float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dmean2D_out,
    float* grad_accum, float* denom, void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera,
    int antialiasing, const float* dL_dalpha, const float* dL_dinvdepth) {
    const char* entry = __func__;
    if (!dL_dalpha || !dL_dinvdepth) return Api(entry).invalid("NULL dL_dalpha / dL_dinvdepth");
    FeatureRows feat;
    if (const int rc = feature_rows(Api(entry), C, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype,
                                    feat, true))
        return rc;
    if (antialiasing && P > 0 && overlaps({dL_dopacity, (size_t)P * 4}, {{dL_dmean2D_out, (size_t)P * 3 * 4}}))
        return Api(entry).invalid("dL_dopacity overlaps another output");
    const auto run = [&](auto map, float scale) {
        return backward_accum_impl(entry, P, D, M, R, C, background, width, height, means3D, shs, colors_precomp,
                                   scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos,
                                   tan_fovx, tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, map,
                                   scale, dL_depths, scratch, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature,
                                   dL_dmean3D, dL_dcov3D_precomp, dL_dsh, dL_dscale, dL_drot, dL_dmean2D_out,
                                   grad_accum, denom, composite_done_event, debug, cuda_stream, false, dL_dcamera,
                                   feat, antialiasing != 0, dL_dalpha, dL_dinvdepth);
    };
    if (dL_dfeaturepix_dtype == F3DGS_F16)
        return run(static_cast<const __half*>(dL_dfeaturepix), dL_dfeaturepix_scale);
    return run(static_cast<const float*>(dL_dfeaturepix), 1.f);
}

}  // extern "C"

namespace {
// Shared body of f3dgs_lift_features_accum (TF = float) and f3dgs_lift_features_accum_f16 (TF = __half, the map only).
template <typename TF>
int lift_impl(const char* entry, int P, int R, int C, int width, int height, char* geom_buffer, char* binning_buffer,
              char* image_buffer, const TF* feature_map, float* feature_sum, float* weight_sum, void* cuda_stream) {
    const Api api(entry);
    if (P < 0 || R < 0 || width <= 0 || height <= 0 || C < 1 || C > F3DGS_MAX_FEATURE_DIM)
        return api.invalid("bad sizes (P >= 0, R >= 0, width, height >= 1, 1 <= C <= F3DGS_MAX_FEATURE_DIM)");
    if (P == 0 || R == 0) return 0;  // nothing is blended (a forward with R == 0 may leave an empty binning buffer)
    if (!geom_buffer || !binning_buffer || !image_buffer) return api.invalid("missing forward buffers");
    if (!feature_map || !feature_sum || !weight_sum) return api.invalid("NULL pointer (feature_map, feature_sum or weight_sum)");
    // both kernels reduce into the outputs while other warps still read the map
    const Range rmap{feature_map, (size_t)C * width * height * sizeof(TF)}, rws{weight_sum, (size_t)P * 4};
    if (overlaps({feature_sum, (size_t)P * C * 4}, {rmap, rws}) || overlaps(rws, {rmap}))
        return api.invalid("feature_sum, weight_sum and feature_map must not overlap");

    const ViewParams vp = make_view(P, 0, 0, C, width, height, 0.f, 0.f, 1.f, nullptr, nullptr, nullptr);
    const cudaError_t e = launch_feature_lift(vp, forward_buffers(vp, R, geom_buffer, binning_buffer, image_buffer),
                                              feature_map, feature_sum, weight_sum, (cudaStream_t)cuda_stream);
    return composite_bwd_result(api, e, "lift launch");
}
}  // namespace

extern "C" {

int f3dgs_lift_features_accum(int P, int R, int C, int width, int height, char* geom_buffer, char* binning_buffer,
                              char* image_buffer, const float* feature_map, float* feature_sum, float* weight_sum,
                              void* cuda_stream) {
    return lift_impl(__func__, P, R, C, width, height, geom_buffer, binning_buffer, image_buffer, feature_map,
                     feature_sum, weight_sum, cuda_stream);
}

int f3dgs_lift_features_accum_f16(int P, int R, int C, int width, int height, char* geom_buffer, char* binning_buffer,
                                  char* image_buffer, const uint16_t* feature_map, float* feature_sum, float* weight_sum,
                                  void* cuda_stream) {
    return lift_impl(__func__, P, R, C, width, height, geom_buffer, binning_buffer, image_buffer,
                     reinterpret_cast<const __half*>(feature_map), feature_sum, weight_sum, cuda_stream);
}

}  // extern "C"

namespace {
// The float16 entry points (_f16gt, _f16, _f16x) validate and launch as their float32 twins do.  Half data is IEEE
// binary16 bits at the ABI (uint16_t) and __half in the kernels.
template <typename FM, typename GT>
int feature_resize_fwd_impl(const char* entry, int C, int H, int W, int Hg, int Wg, const FM* feature_map,
                            const GT* gt, float grad_scale, float* out, float* loss_sum, void* cuda_stream) {
    const Api api(entry);
    if (C < 0 || H <= 0 || W <= 0 || Hg <= 0 || Wg <= 0) return api.invalid("bad sizes");
    if (C == 0) return 0;
    if (!feature_map || !out) return api.invalid("NULL pointer");
    if constexpr (std::is_same_v<GT, __half> || std::is_same_v<FM, __half>) {
        // a float16 target is required (no target is the _f16 symbol's job for a float16 map, the float32 one's
        // otherwise); out's 4-byte elements cannot alias 2-byte ones element for element
        if (std::is_same_v<GT, __half> && !gt) return api.invalid("NULL pointer (gt is required)");
        const size_t n = (size_t)C * Hg * Wg;
        if (overlaps({out, n * 4}, {{feature_map, (size_t)C * H * W * sizeof(FM)}, {gt, n * sizeof(GT)}}))
            return api.invalid("out overlaps feature_map or gt");
    }
    return api.cuda(launch_feature_resize_fwd(C, H, W, Hg, Wg, feature_map, gt, grad_scale, out, loss_sum,
                                              (cudaStream_t)cuda_stream));
}
}  // namespace

extern "C" {

int f3dgs_feature_resize_fwd(int C, int H, int W, int Hg, int Wg, const float* feature_map, const float* gt,
                             float grad_scale, float* out, float* loss_sum, void* cuda_stream) {
    return feature_resize_fwd_impl(__func__, C, H, W, Hg, Wg, feature_map, gt, grad_scale, out, loss_sum, cuda_stream);
}

int f3dgs_feature_resize_fwd_f16gt(int C, int H, int W, int Hg, int Wg, const float* feature_map, const uint16_t* gt,
                                   float grad_scale, float* out, float* loss_sum, void* cuda_stream) {
    return feature_resize_fwd_impl(__func__, C, H, W, Hg, Wg, feature_map, reinterpret_cast<const __half*>(gt),
                                   grad_scale, out, loss_sum, cuda_stream);
}

int f3dgs_feature_resize_fwd_f16(int C, int H, int W, int Hg, int Wg, const uint16_t* feature_map, const float* gt,
                                 float grad_scale, float* out, float* loss_sum, void* cuda_stream) {
    return feature_resize_fwd_impl(__func__, C, H, W, Hg, Wg, reinterpret_cast<const __half*>(feature_map), gt,
                                   grad_scale, out, loss_sum, cuda_stream);
}

int f3dgs_feature_resize_fwd_f16_f16gt(int C, int H, int W, int Hg, int Wg, const uint16_t* feature_map,
                                       const uint16_t* gt, float grad_scale, float* out, float* loss_sum,
                                       void* cuda_stream) {
    return feature_resize_fwd_impl(__func__, C, H, W, Hg, Wg, reinterpret_cast<const __half*>(feature_map),
                                   reinterpret_cast<const __half*>(gt), grad_scale, out, loss_sum, cuda_stream);
}

int f3dgs_feature_resize_bwd(int C, int H, int W, int Hg, int Wg, const float* dout, float* dL_dfeature_map,
                             void* cuda_stream) {
    const Api api(__func__);
    if (C < 0 || H <= 0 || W <= 0 || Hg <= 0 || Wg <= 0) return api.invalid("bad sizes");
    if (C == 0) return 0;
    if (!dout || !dL_dfeature_map) return api.invalid("NULL pointer");
    return api.cuda(
        launch_feature_resize_bwd(C, H, W, Hg, Wg, dout, dL_dfeature_map, 1.f, (cudaStream_t)cuda_stream));
}

int f3dgs_feature_resize_bwd_f16(int C, int H, int W, int Hg, int Wg, const float* dout, float out_scale,
                                 uint16_t* dL_dfeature_map, void* cuda_stream) {
    const Api api(__func__);
    if (C < 0 || H <= 0 || W <= 0 || Hg <= 0 || Wg <= 0) return api.invalid("bad sizes");
    if (C == 0) return 0;
    if (!dout || !dL_dfeature_map) return api.invalid("NULL pointer");
    if (!std::isfinite(out_scale) || out_scale == 0.f) return api.invalid("out_scale must be finite and nonzero");
    // the gather reads dout around every element it writes
    if (overlaps({dL_dfeature_map, (size_t)C * H * W * 2}, {{dout, (size_t)C * Hg * Wg * 4}}))
        return api.invalid("dL_dfeature_map overlaps dout");
    return api.cuda(launch_feature_resize_bwd(C, H, W, Hg, Wg, dout, reinterpret_cast<__half*>(dL_dfeature_map),
                                              out_scale, (cudaStream_t)cuda_stream));
}

int f3dgs_image_loss(int planes, int H, int W, const float* image, const float* gt, float w_l1, float w_ssim, float* sums,
                     float* dL_dimage, void* cuda_stream) {
    const Api api(__func__);
    if (planes < 0 || H <= 0 || W <= 0) return api.invalid("bad sizes");
    if (planes == 0) return 0;
    if (!image_loss_grid_ok(planes, H, W)) return api.invalid("sizes exceed the launch grid limits");
    if (!image || !gt || !sums) return api.invalid("NULL pointer");
    // a CTA reads its neighbours' pixels (the window halo), so the gradient cannot overwrite an input
    const size_t n = (size_t)planes * H * W * sizeof(float);
    if (overlaps({dL_dimage, n}, {{image, n}, {gt, n}})) return api.invalid("dL_dimage overlaps image or gt");
    return api.cuda(launch_image_loss(planes, H, W, image, gt, w_l1, w_ssim, sums, dL_dimage, (cudaStream_t)cuda_stream));
}

}  // extern "C"

namespace {
template <typename Y>
int decoder_forward_impl(const char* entry, int Cin, int Cout, int N, const float* weight, const float* bias,
                         const float* x, Y* y, void* cuda_stream) {
    const Api api(entry);
    if (Cin < 1 || Cin > kDecoderMaxCin || Cout < 1 || Cout > kDecoderMaxCout || N < 1)
        return api.invalid("bad sizes (1 <= Cin <= 256, 1 <= Cout <= 4096, N >= 1)");
    if (!decoder_grid_ok(Cin, Cout, N)) return api.invalid("sizes exceed the launch grid limits");
    if (!weight || !x || !y) return api.invalid("NULL pointer");
    if (overlaps({y, (size_t)Cout * N * sizeof(Y)},
                 {{weight, (size_t)Cout * Cin * 4}, {bias, (size_t)Cout * 4}, {x, (size_t)Cin * N * 4}}))
        return api.invalid("y overlaps an input");
    return api.cuda(launch_decoder_forward(Cin, Cout, N, weight, bias, x, y, (cudaStream_t)cuda_stream));
}

template <typename GT>
int decoder_l1_impl(const char* entry, int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                    const GT* gt, float grad_scale, float* loss_sum, float* dL_dx, float* dL_dweight, float* dL_dbias,
                    void* cuda_stream) {
    const Api api(entry);
    if (Cin < 1 || Cin > kDecoderMaxCin || Cout < 1 || Cout > kDecoderMaxCout || N < 1)
        return api.invalid("bad sizes (1 <= Cin <= 256, 1 <= Cout <= 4096, N >= 1)");
    if (!decoder_grid_ok(Cin, Cout, N)) return api.invalid("sizes exceed the launch grid limits");
    if (!weight || !x || !gt || !loss_sum || !dL_dx || !dL_dweight) return api.invalid("NULL pointer");
    if ((bias == nullptr) != (dL_dbias == nullptr)) return api.invalid("NULL pointer (dL_dbias goes with bias)");
    const size_t nx = (size_t)Cin * N * 4, nw = (size_t)Cout * Cin * 4, nb = (size_t)Cout * 4;
    // a warp reads x of its own pixels only, but kernel B reads all of x after dL_dx is written
    if (overlaps({dL_dx, nx}, {{x, nx}, {gt, (size_t)Cout * N * sizeof(GT)}, {weight, nw}, {bias, nb},
                               {dL_dweight, nw}, {dL_dbias, nb}}))
        return api.invalid("dL_dx overlaps an input");
    return api.cuda(launch_decoder_l1(Cin, Cout, N, weight, bias, x, gt, grad_scale, loss_sum, dL_dx, dL_dweight,
                                      dL_dbias, (cudaStream_t)cuda_stream));
}

template <typename X>
int feature_query_impl(const char* entry, int C, int D, int K, int N, const float* weight, const float* bias, const X* x,
                       const float* text, float logit_scale, const uint8_t* positive, int64_t* labels, float* prob,
                       float* logits, void* cuda_stream) {
    const Api api(entry);
    if (K < 1 || K > kQueryMaxK || D < 1 || D > kQueryMaxD || C < 1 || N < 0 || (weight && C > kDecoderMaxCin))
        return api.invalid("bad sizes (1 <= K <= 256, 1 <= D <= 4096, N >= 0, 1 <= C <= 256 with a decoder)");
    if (!weight && D != C) return api.invalid("D != C needs a decoder weight");
    if (bias && !weight) return api.invalid("bias without weight");
    if (!x || !text) return api.invalid("NULL pointer (x and text are required)");
    if (!labels && !prob && !logits) return api.invalid("no output requested");
    if (prob && !positive) return api.invalid("prob needs a positive set");
    if (!std::isfinite(logit_scale)) return api.invalid("logit_scale is not finite");
    const size_t n = (size_t)N;
    const Range in[] = {{weight, (size_t)D * C * 4}, {bias, (size_t)D * 4}, {x, (size_t)C * n * sizeof(X)},
                        {text, (size_t)K * D * 4}, {positive, (size_t)K}};
    const Range out[] = {{labels, n * 8}, {prob, n * 4}, {logits, (size_t)K * n * 4}};
    for (int i = 0; i < 3; i++) {
        if (overlaps(out[i], in)) return api.invalid("an output overlaps an input");
        for (int j = 0; j < i; j++)
            if (overlaps(out[i], {out[j]})) return api.invalid("outputs overlap");
    }
    return api.cuda(launch_feature_query(C, D, K, N, weight, bias, x, text, logit_scale, positive, labels, prob, logits,
                                         (cudaStream_t)cuda_stream));
}

// ---- feature PCA: shared validation of (C, N)
bool pca_sizes_ok(int C, int N) { return C >= kPcaMinC && C <= kPcaMaxC && N >= 7; }  // n = ceil(N / 3) >= 3

template <typename X>
int pca_moments_impl(const char* entry, int C, int N, const X* x, char* scratch, float* mean, double* cov,
                     void* cuda_stream) {
    const Api api(entry);
    if (!pca_sizes_ok(C, N)) return api.invalid("bad sizes (3 <= C <= 1024, N >= 7)");
    if (!x || !scratch || !mean || !cov) return api.invalid("NULL pointer");
    const Range rx{x, (size_t)C * N * sizeof(X)}, rs{scratch, pca_scratch_fixed_bytes(C, N)};
    const Range rm{mean, (size_t)C * 4}, rc{cov, (size_t)C * C * 8};
    if (overlaps(rs, {rx}) || overlaps(rm, {rx, rs}) || overlaps(rc, {rx, rs, rm}))
        return api.invalid("scratch, mean and cov must not overlap x or each other");
    return api.cuda(launch_pca_moments(C, N, x, scratch, mean, cov, (cudaStream_t)cuda_stream));
}

template <typename X>
int pca_range_impl(const char* entry, int C, int N, const X* x, const float* mean, const float* components, char* scratch,
                   float* range, void* cuda_stream) {
    const Api api(entry);
    if (!pca_sizes_ok(C, N)) return api.invalid("bad sizes (3 <= C <= 1024, N >= 7)");
    if (!x || !mean || !components || !scratch || !range) return api.invalid("NULL pointer");
    const Range rx{x, (size_t)C * N * sizeof(X)}, rm{mean, (size_t)C * 4}, rc{components, (size_t)3 * C * 4};
    const Range rs{scratch, pca_scratch_fixed_bytes(C, N)}, rr{range, 8};
    if (overlaps(rs, {rx, rm, rc}) || overlaps(rr, {rx, rm, rc, rs}))
        return api.invalid("scratch or range overlaps an input");
    size_t sb = 0;
    CUDA_TRY(pca_scratch_bytes(C, N, &sb));  // the sort's share of the scratch is sized by CUB for the current device
    if (overlaps({scratch, sb}, {rx, rm, rc, rr})) return api.invalid("scratch or range overlaps an input");
    return api.cuda(launch_pca_range(C, N, x, mean, components, scratch, range, (cudaStream_t)cuda_stream));
}

template <typename X>
int pca_image_impl(const char* entry, int C, int N, const X* x, const float* mean, const float* components,
                   const float* range, float* image, void* cuda_stream) {
    const Api api(entry);
    if (!pca_sizes_ok(C, N)) return api.invalid("bad sizes (3 <= C <= 1024, N >= 7)");
    if (!x || !mean || !components || !range || !image) return api.invalid("NULL pointer");
    if (overlaps({image, (size_t)N * 3 * 4}, {{x, (size_t)C * N * sizeof(X)}, {mean, (size_t)C * 4},
                                              {components, (size_t)3 * C * 4}, {range, 8}}))
        return api.invalid("image overlaps an input");
    return api.cuda(launch_pca_image(C, N, x, mean, components, range, image, (cudaStream_t)cuda_stream));
}

// Body of the *_scratch_bytes entry points: `query` sizes the scratch; 0, with the last error set, if it fails.
template <typename Query>
size_t scratch_bytes(const char* entry, Query query) {
    const Api api(entry);
    size_t bytes = 0;
    return api.cuda(query(&bytes)) == 0 ? bytes : 0;
}
}  // namespace

extern "C" {

int f3dgs_decoder_forward(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x, float* y,
                          void* cuda_stream) {
    return decoder_forward_impl(__func__, Cin, Cout, N, weight, bias, x, y, cuda_stream);
}

int f3dgs_decoder_forward_f16(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                              uint16_t* y, void* cuda_stream) {
    return decoder_forward_impl(__func__, Cin, Cout, N, weight, bias, x, reinterpret_cast<__half*>(y), cuda_stream);
}

int f3dgs_decoder_l1(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x, const float* gt,
                     float grad_scale, float* loss_sum, float* dL_dx, float* dL_dweight, float* dL_dbias,
                     void* cuda_stream) {
    return decoder_l1_impl(__func__, Cin, Cout, N, weight, bias, x, gt, grad_scale, loss_sum, dL_dx, dL_dweight,
                           dL_dbias, cuda_stream);
}

int f3dgs_decoder_l1_f16gt(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                           const uint16_t* gt, float grad_scale, float* loss_sum, float* dL_dx, float* dL_dweight,
                           float* dL_dbias, void* cuda_stream) {
    return decoder_l1_impl(__func__, Cin, Cout, N, weight, bias, x, reinterpret_cast<const __half*>(gt), grad_scale,
                           loss_sum, dL_dx, dL_dweight, dL_dbias, cuda_stream);
}

int f3dgs_feature_query(int C, int D, int K, int N, const float* weight, const float* bias, const float* x,
                        const float* text, float logit_scale, const uint8_t* positive, int64_t* labels, float* prob,
                        float* logits, void* cuda_stream) {
    return feature_query_impl(__func__, C, D, K, N, weight, bias, x, text, logit_scale, positive, labels, prob, logits,
                              cuda_stream);
}

int f3dgs_feature_query_f16x(int C, int D, int K, int N, const float* weight, const float* bias, const uint16_t* x,
                             const float* text, float logit_scale, const uint8_t* positive, int64_t* labels,
                             float* prob, float* logits, void* cuda_stream) {
    return feature_query_impl(__func__, C, D, K, N, weight, bias, reinterpret_cast<const __half*>(x), text, logit_scale,
                              positive, labels, prob, logits, cuda_stream);
}

size_t f3dgs_feature_pca_scratch_bytes(int C, int N) {
    return scratch_bytes(__func__,
                         [=](size_t* b) { return pca_sizes_ok(C, N) ? pca_scratch_bytes(C, N, b) : cudaSuccess; });
}

int f3dgs_feature_pca_moments(int C, int N, const float* x, char* scratch, float* mean, double* cov, void* cuda_stream) {
    return pca_moments_impl(__func__, C, N, x, scratch, mean, cov, cuda_stream);
}

int f3dgs_feature_pca_moments_f16x(int C, int N, const uint16_t* x, char* scratch, float* mean, double* cov,
                                   void* cuda_stream) {
    return pca_moments_impl(__func__, C, N, reinterpret_cast<const __half*>(x), scratch, mean, cov, cuda_stream);
}

int f3dgs_feature_pca_range(int C, int N, const float* x, const float* mean, const float* components, char* scratch,
                            float* range, void* cuda_stream) {
    return pca_range_impl(__func__, C, N, x, mean, components, scratch, range, cuda_stream);
}

int f3dgs_feature_pca_range_f16x(int C, int N, const uint16_t* x, const float* mean, const float* components,
                                 char* scratch, float* range, void* cuda_stream) {
    return pca_range_impl(__func__, C, N, reinterpret_cast<const __half*>(x), mean, components, scratch, range,
                          cuda_stream);
}

int f3dgs_feature_pca_image(int C, int N, const float* x, const float* mean, const float* components,
                            const float* range, float* image, void* cuda_stream) {
    return pca_image_impl(__func__, C, N, x, mean, components, range, image, cuda_stream);
}

int f3dgs_feature_pca_image_f16x(int C, int N, const uint16_t* x, const float* mean, const float* components,
                                 const float* range, float* image, void* cuda_stream) {
    return pca_image_impl(__func__, C, N, reinterpret_cast<const __half*>(x), mean, components, range, image,
                          cuda_stream);
}

size_t f3dgs_knn_scratch_bytes(int P) {
    return scratch_bytes(__func__, [=](size_t* b) { return knn_scratch_bytes(P, b); });
}

int f3dgs_knn_mean_dist(int P, const float* points, float* out, char* scratch, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0) return api.invalid("P < 0");
    if (P == 0) return 0;
    if (!points || !out || !scratch) return api.invalid("NULL pointer");
    const Range ro{out, (size_t)P * 4};
    if (overlaps(ro, {{points, (size_t)P * 12}, {scratch, knn_scratch_fixed_bytes(P)}}))
        return api.invalid("out overlaps points or scratch");
    size_t sb = 0;
    CUDA_TRY(knn_scratch_bytes(P, &sb));  // the sort's share of the scratch is sized by CUB for the current device
    if (overlaps(ro, {{scratch, sb}})) return api.invalid("out overlaps points or scratch");
    return api.cuda(launch_knn_mean_dist(P, points, out, scratch, (cudaStream_t)cuda_stream));
}

size_t f3dgs_densify_scratch_bytes(int P) {
    return scratch_bytes(__func__, [=](size_t* b) { return densify_scratch_bytes(P, b); });
}

int f3dgs_densify_plan(int P, const float* grad_accum, const float* denom, const float* raw_opacity,
                       const float* raw_scaling, float max_grad, float dense_scale, float min_opacity,
                       float max_world_scale, char* scratch, int32_t* counts, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || 3 * (long long)P > INT_MAX) return api.invalid("bad sizes (0 <= 3 P <= INT_MAX)");
    if (!counts || (P > 0 && (!grad_accum || !denom || !raw_opacity || !raw_scaling || !scratch)))
        return api.invalid("NULL pointer");
    if (overlaps({counts, 16}, {{scratch, densify_scratch_fixed_bytes(P)}}))
        return api.invalid("counts overlaps scratch");
    return api.cuda(launch_densify_plan(P, grad_accum, denom, raw_opacity, raw_scaling, max_grad, dense_scale,
                                        min_opacity, max_world_scale, scratch, counts, (cudaStream_t)cuda_stream));
}

int f3dgs_densify_apply(int P, int M, int C, const char* scratch, const int32_t counts[4], const float* normals,
                        const f3dgs_gaussian_fields src[3], const f3dgs_gaussian_fields dst[3], void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || 3 * (long long)P > INT_MAX || M < 1 || C < 0 || C > F3DGS_MAX_FEATURE_DIM)
        return api.invalid("bad sizes (0 <= 3 P <= INT_MAX, M >= 1, 0 <= C <= F3DGS_MAX_FEATURE_DIM)");
    if (!counts || !src || !dst) return api.invalid("NULL pointer");
    const long long A = counts[0], B = counts[1], Cc = counts[2], Ns = counts[3], Pn = A + B + 2 * Cc;
    if (A < 0 || B < 0 || Cc < 0 || A > P || B > P || Cc > Ns || Ns > P || 3 * Pn > INT_MAX)
        return api.invalid("counts are not those of a plan over P Gaussians");
    if (Ns > 0 && !normals) return api.invalid("NULL pointer (normals)");
    if (P > 0 && !scratch) return api.invalid("NULL pointer (scratch)");
    const size_t width[7] = {3, 3, 3 * (size_t)(M - 1), 1, 3, 4, (size_t)C};
    const float* s[21];
    float* d[21];
    for (int g = 0; g < 3; g++) {
        const f3dgs_gaussian_fields* f[2] = {&src[g], &dst[g]};
        for (int k = 0; k < 2; k++) {
            const float* p[7] = {f[k]->xyz, f[k]->f_dc, f[k]->f_rest, f[k]->opacity, f[k]->scaling, f[k]->rotation,
                                 f[k]->semantic_feature};
            for (int j = 0; j < 7; j++) {
                if (width[j] && (k ? Pn : P) > 0 && !p[j]) return api.invalid("NULL pointer (a src or dst field)");
                if (k) d[7 * g + j] = const_cast<float*>(p[j]);
                else s[7 * g + j] = p[j];
            }
        }
    }
    Range in[23] = {{scratch, densify_scratch_fixed_bytes(P)}, {normals, (size_t)Ns * 24}};
    for (int j = 0; j < 21; j++) in[2 + j] = {s[j], (size_t)P * width[j % 7] * 4};
    for (int i = 0; i < 21; i++)
        if (overlaps({d[i], (size_t)Pn * width[i % 7] * 4}, in))
            return api.invalid("a dst field overlaps a src field, normals or scratch");
    return api.cuda(launch_densify_apply(P, M, C, scratch, counts, normals, s, d, (cudaStream_t)cuda_stream));
}

int f3dgs_reset_opacity(int P, float* raw_opacity, float* exp_avg, float* exp_avg_sq, float ceiling, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0) return api.invalid("P < 0");
    if (P == 0) return 0;
    if (!raw_opacity || !exp_avg || !exp_avg_sq) return api.invalid("NULL pointer");
    return api.cuda(launch_reset_opacity(P, raw_opacity, exp_avg, exp_avg_sq, ceiling, (cudaStream_t)cuda_stream));
}

int f3dgs_activate(int P, int M, const float* raw_opacity, const float* raw_scaling, const float* raw_rotation,
                   const float* features_dc, const float* features_rest, float* opacity, float* scales, float* rotations,
                   float* shs, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || M < 0) return api.invalid("bad sizes (P < 0 or M < 0)");
    if (P == 0) return 0;
    if ((raw_opacity && !opacity) || (raw_scaling && !scales) || (raw_rotation && !rotations) ||
        (features_dc && (!shs || M < 1 || (M > 1 && !features_rest))))
        return api.invalid("NULL pointer (an input without its output, or features_dc without shs, M >= 1 and, for "
                           "M > 1, features_rest)");
    return api.cuda(launch_activate(P, M, raw_opacity, raw_scaling, raw_rotation, features_dc, features_rest, opacity,
                                    scales, rotations, shs, (cudaStream_t)cuda_stream));
}

int f3dgs_adam_step(int kind, size_t n, int M, float* param, const float* grad_activated, float* exp_avg, float* exp_avg_sq,
                    float lr, float beta1, float beta2, float eps, int step, void* cuda_stream) {
    const Api api(__func__);
    if (kind < F3DGS_PARAM_IDENTITY || kind > F3DGS_PARAM_SH_REST) return api.invalid("unknown parameter kind");
    if (step < 1) return api.invalid("step < 1");
    if (!param || !grad_activated || !exp_avg || !exp_avg_sq) return api.invalid("NULL pointer");
    if (kind == F3DGS_PARAM_NORMALIZE4 && (n % 4 != 0)) return api.invalid("n % 4 != 0 for F3DGS_PARAM_NORMALIZE4");
    if ((kind == F3DGS_PARAM_SH_DC || kind == F3DGS_PARAM_SH_REST) && M < (kind == F3DGS_PARAM_SH_REST ? 2 : 1))
        return api.invalid("M < 1 for F3DGS_PARAM_SH_DC or M < 2 for F3DGS_PARAM_SH_REST");
    if (n == 0) return 0;
    return api.cuda(launch_adam_step(kind, n, M, param, grad_activated, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, step,
                                     (cudaStream_t)cuda_stream));
}

int f3dgs_adam_step_f16out(int kind, size_t n, int M, float* param, const float* grad_activated, float* exp_avg,
                           float* exp_avg_sq, uint16_t* param_f16, float lr, float beta1, float beta2, float eps,
                           int step, void* cuda_stream) {
    const Api api(__func__);
    if (kind != F3DGS_PARAM_IDENTITY) return api.invalid("kind must be F3DGS_PARAM_IDENTITY");
    if (step < 1) return api.invalid("step < 1");
    if (!param || !grad_activated || !exp_avg || !exp_avg_sq || !param_f16) return api.invalid("NULL pointer");
    if (overlaps({param_f16, n * 2}, {{param, n * 4}, {grad_activated, n * 4}, {exp_avg, n * 4}, {exp_avg_sq, n * 4}}))
        return api.invalid("param_f16 overlaps param, grad_activated, exp_avg or exp_avg_sq");
    if (n == 0) return 0;
    return api.cuda(launch_adam_step(kind, n, M, param, grad_activated, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, step,
                                     (cudaStream_t)cuda_stream, reinterpret_cast<__half*>(param_f16)));
}

int f3dgs_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                       uint8_t* present, void* cuda_stream) {
    (void)projmatrix;  // the reference's frustum side test is commented out (auxiliary.h:160)
    const Api api(__func__);
    if (P < 0) return api.invalid("P < 0");
    if (P == 0) return 0;
    if (!means3D || !viewmatrix || !present) return api.invalid("NULL pointer");
    launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)cuda_stream);
    return api.cuda(cudaGetLastError());
}

}  // extern "C"
