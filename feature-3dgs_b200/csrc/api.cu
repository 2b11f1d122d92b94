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
#include <initializer_list>
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

// Does the output range `out` share a byte with any of the ranges `in` other than itself (`out` may be one of them)?
template <size_t N>
bool overlaps(const Range& out, const Range (&in)[N]) {
    for (const Range& r : in) {
        const uintptr_t x = (uintptr_t)out.p, y = (uintptr_t)r.p;
        if (&r != &out && out.p && r.p && x < y + r.bytes && y < x + out.bytes) return true;
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

// Every dtype code of a typed entry is F3DGS_F32 or F3DGS_F16
int check_dtypes(const Api& api, std::initializer_list<int> codes) {
    for (const int t : codes)
        if (t != F3DGS_F32 && t != F3DGS_F16) return api.invalid("unknown dtype code");
    return 0;
}

// Shared body of f3dgs_forward, f3dgs_forward_f16, f3dgs_forward_antialiased, f3dgs_forward_alpha_invdepth and
// f3dgs_forward_distortion.  semantic_feature and out_feature_map are float16 if f16, else float32.  antialiasing:
// op_eff = opacity * rho in the records.  out_alpha / out_invdepth (f3dgs_forward_alpha_invdepth, which has checked that
// both are given): the composite also writes the opacity and inverse-depth planes.  out_distortion
// (f3dgs_forward_distortion): the composite also writes the depth distortion plane.
int forward_impl(const char* entry, f3dgs_alloc_fn geometry_alloc, void* geometry_ctx, f3dgs_alloc_fn binning_alloc,
                 void* binning_ctx, f3dgs_alloc_fn image_alloc, void* image_ctx, int P, int D, int M, int C,
                 const float* background, int width, int height, const float* means3D, const float* shs,
                 const float* colors_precomp, const void* semantic_feature, const float* opacities, const float* scales,
                 float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                 const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered,
                 float* out_color, void* out_feature_map, float* out_depth, int* radii, int debug, void* cuda_stream,
                 bool f16 = false, bool antialiasing = false, float* out_alpha = nullptr,
                 float* out_invdepth = nullptr, float* out_distortion = nullptr) {
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
    // the composite writes the planes while it writes the other outputs
    const size_t hw4 = (size_t)width * height * 4;
    const Range outs[] = {{out_color, 3 * hw4}, {out_feature_map, (size_t)C * width * height * (f16 ? 2 : 4)},
                          {out_depth, hw4}, {radii, (size_t)P * 4}, {out_alpha, hw4}, {out_invdepth, hw4},
                          {out_distortion, hw4}};
    if (overlaps(outs[4], outs) || overlaps(outs[5], outs))
        return api.invalid("out_alpha / out_invdepth overlap another output");
    if (overlaps(outs[6], outs)) return api.invalid("out_distortion overlaps another output");

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
        if (f16)
            e = launch_composite_fwd(vp, ranges, point_list, rec, static_cast<const __half*>(semantic_feature),
                                     background, final_T, n_contrib, out_color, static_cast<__half*>(out_feature_map),
                                     out_depth, counters, stream, out_alpha, out_invdepth, out_distortion);
        else
            e = launch_composite_fwd(vp, ranges, point_list, rec, static_cast<const float*>(semantic_feature),
                                     background, final_T, n_contrib, out_color, static_cast<float*>(out_feature_map),
                                     out_depth, counters, stream, out_alpha, out_invdepth, out_distortion);
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
                        D, M, C, background, width, height, means3D, shs, colors_precomp, semantic_feature, opacities,
                        scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                        tan_fovy, prefiltered, out_color, out_feature_map, out_depth, radii, debug, cuda_stream, true);
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
    if (const int rc = check_dtypes(Api(__func__), {semantic_feature_dtype})) return rc;
    return forward_impl(__func__, geometry_alloc, geometry_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx, P,
                        D, M, C, background, width, height, means3D, shs, colors_precomp, semantic_feature, opacities,
                        scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                        tan_fovy, prefiltered, out_color, out_feature_map, out_depth, radii, debug, cuda_stream,
                        semantic_feature_dtype == F3DGS_F16, true);
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
    const Api api(__func__);
    if (!out_alpha || !out_invdepth) return api.invalid("NULL out_alpha / out_invdepth");
    if (const int rc = check_dtypes(api, {semantic_feature_dtype})) return rc;
    return forward_impl(__func__, geometry_alloc, geometry_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx, P,
                        D, M, C, background, width, height, means3D, shs, colors_precomp, semantic_feature, opacities,
                        scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                        tan_fovy, prefiltered, out_color, out_feature_map, out_depth, radii, debug, cuda_stream,
                        semantic_feature_dtype == F3DGS_F16, antialiasing != 0, out_alpha, out_invdepth);
}

int f3dgs_forward_distortion(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx, f3dgs_alloc_fn binning_alloc,
                             void* binning_ctx, f3dgs_alloc_fn image_alloc, void* image_ctx, int P, int D, int M,
                             int C, const float* background, int width, int height, const float* means3D,
                             const float* shs, const float* colors_precomp, const void* semantic_feature,
                             int semantic_feature_dtype, const float* opacities, const float* scales,
                             float scale_modifier, const float* rotations, const float* cov3D_precomp,
                             const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                             float tan_fovy, int prefiltered, float* out_color, void* out_feature_map,
                             float* out_depth, int* radii, int debug, void* cuda_stream, int antialiasing,
                             float* out_distortion) {
    const Api api(__func__);
    if (!out_distortion) return api.invalid("NULL out_distortion");
    if (const int rc = check_dtypes(api, {semantic_feature_dtype})) return rc;
    return forward_impl(__func__, geometry_alloc, geometry_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx, P,
                        D, M, C, background, width, height, means3D, shs, colors_precomp, semantic_feature, opacities,
                        scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx,
                        tan_fovy, prefiltered, out_color, out_feature_map, out_depth, radii, debug, cuda_stream,
                        semantic_feature_dtype == F3DGS_F16, antialiasing != 0, nullptr, nullptr, out_distortion);
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

// The map gradient dL_dfeaturepix [C,H,W]: float32, or float16 bits h standing for dL/dO = scale * float(h) (the scale
// is not read for a float32 map)
struct MapGrad {
    const void* p;
    bool f16;
    float scale;
};

// One view's backward, as an entry describes it to `backward`.  An entry initialises the fields up to `stream` from
// its arguments, in f3dgs_backward's order, and the accumulating entries the next group too; every option after that is
// off unless the entry sets it.
struct ViewBackward {
    int P, D, M, R, C;
    const float* background;
    int width, height;
    const float *means3D, *shs, *scales;
    float scale_modifier;
    const float *rotations, *cov3D_precomp, *viewmatrix, *projmatrix, *cam_pos;
    float tan_fovx, tan_fovy;
    const int* radii;
    char *geom_buffer, *binning_buffer, *image_buffer;
    const float* dL_dpix;
    MapGrad map;
    const float* dL_depths;
    float *dL_dmean2D, *dL_dconic, *dL_dopacity, *dL_dcolor, *dL_dsemantic_feature, *dL_dmean3D, *dL_dcov3D, *dL_dsh,
        *dL_dscale, *dL_drot, *dL_dz;
    int debug;
    cudaStream_t stream;

    // The accumulating entries: += into the caller's per-parameter gradient buffers.  Their dL_dmean2D, dL_dconic and
    // dL_dz are NULL and become per-view intermediates in the scratch; so do dL_dcolor and dL_dcov3D, unless they are
    // the gradients of the caller's colors_precomp / cov3D_precomp (which accumulate).
    bool accumulate = false;
    char* scratch = nullptr;
    const float* colors_precomp = nullptr;
    float* dL_dmean2D_out = nullptr;
    float *grad_accum = nullptr, *denom = nullptr;
    cudaEvent_t composite_done = nullptr;

    // the _cam entries' 35 floats, added to
    float* dL_dcamera = nullptr;
    // the Gaussians' features, for the feature term of dL/dalpha
    FeatureRows feat;
    // the forward's records hold op_eff = opacity * rho, so the composite's opacity gradient is dL/dop_eff and the
    // preprocess backward turns it into dL/dopacity (and rho's geometric terms)
    bool antialiasing = false;
    // the gradients of the forward's opacity and inverse-depth planes, added to dL/dalpha and dL/dz by the composite
    const float *dL_dalpha = nullptr, *dL_dinvdepth = nullptr;
    // the _absgrad entries: AbsGS's per-view statistic [P,3] (required there; the accumulating entry zeroes it), and the
    // accumulating entry's grad_accum_abs [P] (optional)
    bool absgrad = false;
    float *dL_dmean2D_abs = nullptr, *grad_accum_abs = nullptr;
    // the _distortion entries: the forward's depth plane and the gradient of its depth distortion, added to dL/dalpha
    // and dL/dz by the composite
    const float *depth = nullptr, *dL_ddistortion = nullptr;
};

// The features of a _feature_geometry, _antialiased or _alpha_invdepth entry, after the checks every such entry makes
// before any other.  `required` (the _feature_geometry entries): C > 0 needs features; otherwise a NULL
// semantic_feature means no feature term.
int feature_rows(const Api& api, ViewBackward& b, const void* semantic_feature, int semantic_feature_dtype,
                 int dL_dfeaturepix_dtype, bool required = false) {
    if (const int rc = check_dtypes(api, {semantic_feature_dtype, dL_dfeaturepix_dtype})) return rc;
    if (b.C > 0 && !semantic_feature && required) return api.invalid("NULL semantic_feature");
    b.feat = {b.C > 0 ? semantic_feature : nullptr, semantic_feature_dtype == F3DGS_F16};
    return 0;
}

// Shared body of every backward entry: f3dgs_backward (the reference's assign-into-zeroed-buffers contract),
// f3dgs_backward_accum (b.accumulate) and their float16, _cam, _feature_geometry, _antialiased and _alpha_invdepth
// twins.  Under antialiasing the assigning backward lets the composite write into dL_dopacity and rescales it in place;
// the accumulating one needs dL/dop_eff of this view alone, so the composite writes into P zeroed floats of the
// device's default memory pool.
int backward(const Api& api, ViewBackward b) {
    const int P = b.P, C = b.C, debug = b.debug;
    const cudaStream_t stream = b.stream;
    if (b.accumulate) {
        if (P <= 0) return P == 0 ? 0 : api.invalid("bad sizes");
        if (!b.scratch) return api.invalid("NULL scratch");
        if ((b.colors_precomp != nullptr) != (b.dL_dcolor != nullptr) ||
            (b.cov3D_precomp != nullptr) != (b.dL_dcov3D != nullptr))
            return api.invalid("dL_dcolors_precomp / dL_dcov3D_precomp go with colors_precomp / cov3D_precomp");
        const ScratchLayout sl((size_t)P);
        const auto in_scratch = [&](size_t offset) { return reinterpret_cast<float*>(b.scratch + offset); };
        b.dL_dmean2D = in_scratch(sl.mean2D);
        b.dL_dconic = in_scratch(sl.conic);
        b.dL_dz = in_scratch(sl.dz);
        if (!b.dL_dcolor) b.dL_dcolor = in_scratch(sl.color);
        if (!b.dL_dcov3D) b.dL_dcov3D = in_scratch(sl.cov3D);
    }
    if (P < 0 || b.width <= 0 || b.height <= 0 || C < 0 || C > F3DGS_MAX_FEATURE_DIM || b.R < 0)
        return api.invalid("bad sizes");
    if (P == 0) return 0;
    if (!b.geom_buffer || !b.binning_buffer || !b.image_buffer) return api.invalid("missing forward buffers");
    if (!b.dL_dpix || !b.dL_depths || (C > 0 && (!b.map.p || !b.dL_dsemantic_feature)) || !b.dL_dmean2D ||
        !b.dL_dconic || !b.dL_dopacity || !b.dL_dcolor || !b.dL_dmean3D || !b.dL_dcov3D || !b.dL_dz)
        return api.invalid("NULL gradient pointer");
    if (b.shs && !b.dL_dsh) return api.invalid("shs given but dL_dsh NULL");
    if (b.scales && (!b.rotations || !b.dL_dscale || !b.dL_drot))
        return api.invalid("scales given but rotations/dL_dscale/dL_drot NULL");
    if ((b.grad_accum == nullptr) != (b.denom == nullptr)) return api.invalid("grad_accum and denom go together");
    if (b.absgrad && !b.dL_dmean2D_abs) return api.invalid("NULL dL_dmean2D_abs");
    if (b.grad_accum_abs && !b.grad_accum) return api.invalid("grad_accum_abs needs grad_accum and denom");
    if (b.map.f16) {
        if (!std::isfinite(b.map.scale) || b.map.scale == 0.f)
            return api.invalid("dL_dfeaturepix_scale must be finite and nonzero");
        // the feature kernel reduces into dL_dsemantic_feature while other warps still read the map
        if (overlaps({b.dL_dsemantic_feature, (size_t)P * C * 4}, {{b.map.p, (size_t)C * b.width * b.height * 2}}))
            return api.invalid("dL_dsemantic_feature overlaps dL_dfeaturepix");
    }
    // Every output; an absent one is NULL.  The optional operands are read or written while the kernels write these,
    // so none may overlap an output other than itself.
    const size_t p4 = (size_t)P * 4, hw4 = (size_t)b.width * b.height * 4;
    const size_t scratch_bytes = b.accumulate ? ScratchLayout((size_t)P).bytes : 0;
    const Range outs[] = {{b.dL_dmean2D, 3 * p4}, {b.dL_dconic, 4 * p4}, {b.dL_dopacity, p4}, {b.dL_dcolor, 3 * p4},
                          {b.dL_dsemantic_feature, (size_t)C * p4}, {b.dL_dmean3D, 3 * p4}, {b.dL_dcov3D, 6 * p4},
                          {b.dL_dsh, (size_t)b.M * 3 * p4}, {b.dL_dscale, 3 * p4}, {b.dL_drot, 4 * p4},
                          {b.dL_dz, p4}, {b.grad_accum, p4}, {b.denom, p4},
                          {b.dL_dcamera, F3DGS_CAMERA_GRAD_FLOATS * sizeof(float)}, {b.scratch, scratch_bytes},
                          {b.dL_dmean2D_out, 3 * p4}, {b.dL_dmean2D_abs, 3 * p4}, {b.grad_accum_abs, p4}};
    const Range &opacity = outs[2], &camera = outs[13], &mean2D_abs = outs[16], &accum_abs = outs[17];
    if (overlaps(accum_abs, outs)) return api.invalid("grad_accum_abs overlaps another output");
    if (overlaps(mean2D_abs, outs)) return api.invalid("dL_dmean2D_abs overlaps another output");
    if (overlaps(camera, outs)) return api.invalid("dL_dcamera overlaps another output");
    if (overlaps({b.feat.rows, (size_t)P * C * (b.feat.f16 ? 2 : 4)}, outs))
        return api.invalid("semantic_feature overlaps an output");
    // the preprocess backward writes dL_dopacity under antialiasing
    if (b.antialiasing && overlaps(opacity, outs)) return api.invalid("dL_dopacity overlaps another output");
    if (overlaps({b.dL_dalpha, hw4}, outs) || overlaps({b.dL_dinvdepth, hw4}, outs))
        return api.invalid("dL_dalpha / dL_dinvdepth overlap an output");
    if (overlaps({b.depth, hw4}, outs) || overlaps({b.dL_ddistortion, hw4}, outs))
        return api.invalid("depth / dL_ddistortion overlap an output");
    if (b.accumulate) CUDA_TRY(cudaMemsetAsync(b.scratch, 0, scratch_bytes, stream));
    if (b.accumulate && b.dL_dmean2D_abs) CUDA_TRY(cudaMemsetAsync(b.dL_dmean2D_abs, 0, 3 * p4, stream));

    const ViewParams vp = make_view(P, b.D, b.M, C, b.width, b.height, b.tan_fovx, b.tan_fovy, b.scale_modifier,
                                    b.viewmatrix, b.projmatrix, b.cam_pos);
    const GeomLayout gl((size_t)P);
    const float* cov3d = b.cov3D_precomp ? b.cov3D_precomp : reinterpret_cast<const float*>(b.geom_buffer + gl.cov3d);
    const uint8_t* clamped = reinterpret_cast<const uint8_t*>(b.geom_buffer + gl.clamped);
    const int* radii = b.radii ? b.radii : reinterpret_cast<const int*>(b.geom_buffer + gl.radii);

    cudaError_t e;
    // where the composite puts the opacity gradient: dL/dop_eff under antialiasing (see above)
    struct PoolFloats {  // returned to the pool on every exit
        float* p = nullptr;
        cudaStream_t s;
        ~PoolFloats() {
            if (p) cudaFreeAsync(p, s);
        }
    } op_eff_grad{nullptr, stream};
    float* dL_dop_eff = b.dL_dopacity;
    if (b.antialiasing && b.accumulate) {
        e = cudaMallocAsync((void**)&op_eff_grad.p, (size_t)P * sizeof(float), stream);
        if (e != cudaSuccess)
            return api.fail(F3DGS_ERR_ALLOC, std::string("cudaMallocAsync for dL/dop_eff failed: ") +
                                                 cudaGetErrorString(e));
        CUDA_TRY(cudaMemsetAsync(op_eff_grad.p, 0, (size_t)P * sizeof(float), stream));
        dL_dop_eff = op_eff_grad.p;
    }
    {
        StageTimer t(F3DGS_STAGE_COMPOSITE_BWD, stream);
        const ForwardBuffers fb = forward_buffers(vp, b.R, b.geom_buffer, b.binning_buffer, b.image_buffer);
        const auto composite = [&](auto* dL_dfeaturepix) {
            return launch_composite_bwd(vp, fb, b.background, b.dL_dpix, b.dL_depths, dL_dfeaturepix, b.map.scale,
                                        b.dL_dmean2D, b.dL_dconic, dL_dop_eff, b.dL_dcolor, b.dL_dz,
                                        b.dL_dsemantic_feature, stream, b.feat, b.dL_dalpha, b.dL_dinvdepth,
                                        b.dL_dmean2D_abs, b.depth, b.dL_ddistortion);
        };
        e = b.map.f16 ? composite(static_cast<const __half*>(b.map.p)) : composite(static_cast<const float*>(b.map.p));
    }
    if (const int rc = composite_bwd_result(api, e, "composite_bwd launch")) return rc;
    STAGE_CHECK("composite_bwd");
    // dL_dopacity is final after the composite, or under antialiasing after the preprocess backward
    if (b.composite_done && !b.antialiasing) CUDA_TRY(cudaEventRecord(b.composite_done, stream));
    {
        StageTimer t(F3DGS_STAGE_PREPROCESS_BWD, stream);
        e = launch_preprocess_bwd(vp, b.means3D, radii, b.shs, clamped, b.scales, b.rotations, cov3d, b.dL_dmean2D,
                                  b.dL_dconic, b.dL_dmean3D, b.dL_dcolor, b.dL_dcov3D, b.dL_dsh, b.dL_dscale, b.dL_drot,
                                  b.dL_dz, stream, b.accumulate, b.grad_accum, b.denom, b.dL_dcamera, b.antialiasing,
                                  reinterpret_cast<const SplatRec*>(b.geom_buffer + gl.rec), dL_dop_eff, b.dL_dopacity,
                                  b.dL_dmean2D_abs, b.grad_accum_abs);
    }
    if (e == cudaErrorMemoryAllocation)
        return api.fail(F3DGS_ERR_ALLOC, std::string("cudaMallocAsync for the camera-gradient partials failed: ") +
                                             cudaGetErrorString(e));
    CUDA_TRY(e);
    STAGE_CHECK("preprocess_bwd");
    if (b.composite_done && b.antialiasing) CUDA_TRY(cudaEventRecord(b.composite_done, stream));
    if (b.dL_dmean2D_out)
        CUDA_TRY(cudaMemcpyAsync(b.dL_dmean2D_out, b.dL_dmean2D, (size_t)P * 3 * sizeof(float),
                                 cudaMemcpyDeviceToDevice, stream));
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
    const ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                         cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                         binning_buffer, image_buffer, dL_dpix, {dL_dfeaturepix, false, 1.f}, dL_depths, dL_dmean2D,
                         dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh,
                         dL_dscale, dL_drot, dL_dz, debug, (cudaStream_t)cuda_stream};
    return backward(Api(__func__), b);
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
    const ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                         cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                         binning_buffer, image_buffer, dL_dpix, {dL_dfeaturepix, true, dL_dfeaturepix_scale},
                         dL_depths, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D,
                         dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dz, debug, (cudaStream_t)cuda_stream};
    return backward(Api(__func__), b);
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
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix, {dL_dfeaturepix, false, 1.f}, dL_depths, dL_dmean2D,
                   dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
                   dL_drot, dL_dz, debug, (cudaStream_t)cuda_stream};
    b.dL_dcamera = dL_dcamera;
    return backward(api, b);
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
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix, {dL_dfeaturepix, true, dL_dfeaturepix_scale}, dL_depths,
                   dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh,
                   dL_dscale, dL_drot, dL_dz, debug, (cudaStream_t)cuda_stream};
    b.dL_dcamera = dL_dcamera;
    return backward(api, b);
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
    const ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                         cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                         binning_buffer, image_buffer, dL_dpix, {dL_dfeaturepix, false, 1.f}, dL_depths, nullptr,
                         nullptr, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D,
                         dL_dcov3D_precomp, dL_dsh, dL_dscale, dL_drot, nullptr, debug, (cudaStream_t)cuda_stream,
                         true, scratch, colors_precomp, dL_dmean2D_out, grad_accum, denom,
                         (cudaEvent_t)composite_done_event};
    return backward(Api(__func__), b);
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
    const ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                         cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                         binning_buffer, image_buffer, dL_dpix, {dL_dfeaturepix, true, dL_dfeaturepix_scale},
                         dL_depths, nullptr, nullptr, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature,
                         dL_dmean3D, dL_dcov3D_precomp, dL_dsh, dL_dscale, dL_drot, nullptr, debug,
                         (cudaStream_t)cuda_stream, true, scratch, colors_precomp, dL_dmean2D_out, grad_accum, denom,
                         (cudaEvent_t)composite_done_event};
    return backward(Api(__func__), b);
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
    const Api api(__func__);
    if (!dL_dcamera) return api.invalid("NULL dL_dcamera");
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix, {dL_dfeaturepix, false, 1.f}, dL_depths, nullptr, nullptr,
                   dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D_precomp, dL_dsh,
                   dL_dscale, dL_drot, nullptr, debug, (cudaStream_t)cuda_stream, true, scratch, colors_precomp,
                   dL_dmean2D_out, grad_accum, denom, (cudaEvent_t)composite_done_event};
    b.dL_dcamera = dL_dcamera;
    return backward(api, b);
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
    const Api api(__func__);
    if (!dL_dcamera) return api.invalid("NULL dL_dcamera");
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix, {dL_dfeaturepix, true, dL_dfeaturepix_scale}, dL_depths,
                   nullptr, nullptr, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D,
                   dL_dcov3D_precomp, dL_dsh, dL_dscale, dL_drot, nullptr, debug, (cudaStream_t)cuda_stream, true,
                   scratch, colors_precomp, dL_dmean2D_out, grad_accum, denom, (cudaEvent_t)composite_done_event};
    b.dL_dcamera = dL_dcamera;
    return backward(api, b);
}

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
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, dL_dmean2D,
                   dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
                   dL_drot, dL_dz, debug, (cudaStream_t)cuda_stream};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype, true))
        return rc;
    b.dL_dcamera = dL_dcamera;
    return backward(api, b);
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
    const Api api(__func__);
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, nullptr,
                   nullptr, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D_precomp,
                   dL_dsh, dL_dscale, dL_drot, nullptr, debug, (cudaStream_t)cuda_stream, true, scratch,
                   colors_precomp, dL_dmean2D_out, grad_accum, denom, (cudaEvent_t)composite_done_event};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype, true))
        return rc;
    b.dL_dcamera = dL_dcamera;
    return backward(api, b);
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
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, dL_dmean2D,
                   dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
                   dL_drot, dL_dz, debug, (cudaStream_t)cuda_stream};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype)) return rc;
    b.dL_dcamera = dL_dcamera;
    b.antialiasing = true;
    return backward(api, b);
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
    const Api api(__func__);
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, nullptr,
                   nullptr, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D_precomp,
                   dL_dsh, dL_dscale, dL_drot, nullptr, debug, (cudaStream_t)cuda_stream, true, scratch,
                   colors_precomp, dL_dmean2D_out, grad_accum, denom, (cudaEvent_t)composite_done_event};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype)) return rc;
    b.dL_dcamera = dL_dcamera;
    b.antialiasing = true;
    return backward(api, b);
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
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, dL_dmean2D,
                   dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
                   dL_drot, dL_dz, debug, (cudaStream_t)cuda_stream};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype)) return rc;
    b.dL_dcamera = dL_dcamera;
    b.antialiasing = antialiasing != 0;
    b.dL_dalpha = dL_dalpha;
    b.dL_dinvdepth = dL_dinvdepth;
    return backward(api, b);
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
    const Api api(__func__);
    if (!dL_dalpha || !dL_dinvdepth) return api.invalid("NULL dL_dalpha / dL_dinvdepth");
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, nullptr,
                   nullptr, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D_precomp,
                   dL_dsh, dL_dscale, dL_drot, nullptr, debug, (cudaStream_t)cuda_stream, true, scratch,
                   colors_precomp, dL_dmean2D_out, grad_accum, denom, (cudaEvent_t)composite_done_event};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype)) return rc;
    b.dL_dcamera = dL_dcamera;
    b.antialiasing = antialiasing != 0;
    b.dL_dalpha = dL_dalpha;
    b.dL_dinvdepth = dL_dinvdepth;
    return backward(api, b);
}

int f3dgs_backward_absgrad(int P, int D, int M, int R, int C, const float* background, int width, int height,
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
                           float* dL_dcamera, int antialiasing, const float* dL_dalpha, const float* dL_dinvdepth,
                           float* dL_dmean2D_abs) {
    (void)colors_precomp;
    const Api api(__func__);
    if ((dL_dalpha == nullptr) != (dL_dinvdepth == nullptr)) return api.invalid("dL_dalpha and dL_dinvdepth go together");
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, dL_dmean2D,
                   dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
                   dL_drot, dL_dz, debug, (cudaStream_t)cuda_stream};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype)) return rc;
    b.dL_dcamera = dL_dcamera;
    b.antialiasing = antialiasing != 0;
    b.dL_dalpha = dL_dalpha;
    b.dL_dinvdepth = dL_dinvdepth;
    b.absgrad = true;
    b.dL_dmean2D_abs = dL_dmean2D_abs;
    return backward(api, b);
}

int f3dgs_backward_accum_absgrad(
    int P, int D, int M, int R, int C, const float* background, int width, int height, const float* means3D,
    const float* shs, const float* colors_precomp, const void* semantic_feature, int semantic_feature_dtype,
    const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
    const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
    const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
    const void* dL_dfeaturepix, int dL_dfeaturepix_dtype, float dL_dfeaturepix_scale, const float* dL_depths,
    char* scratch, float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature, float* dL_dmean3D,
    float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dmean2D_out,
    float* grad_accum, float* denom, void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera,
    int antialiasing, const float* dL_dalpha, const float* dL_dinvdepth, float* dL_dmean2D_abs,
    float* grad_accum_abs) {
    const Api api(__func__);
    if ((dL_dalpha == nullptr) != (dL_dinvdepth == nullptr)) return api.invalid("dL_dalpha and dL_dinvdepth go together");
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, nullptr,
                   nullptr, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D_precomp,
                   dL_dsh, dL_dscale, dL_drot, nullptr, debug, (cudaStream_t)cuda_stream, true, scratch,
                   colors_precomp, dL_dmean2D_out, grad_accum, denom, (cudaEvent_t)composite_done_event};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype)) return rc;
    b.dL_dcamera = dL_dcamera;
    b.antialiasing = antialiasing != 0;
    b.dL_dalpha = dL_dalpha;
    b.dL_dinvdepth = dL_dinvdepth;
    b.absgrad = true;
    b.dL_dmean2D_abs = dL_dmean2D_abs;
    b.grad_accum_abs = grad_accum_abs;
    return backward(api, b);
}

int f3dgs_backward_distortion(int P, int D, int M, int R, int C, const float* background, int width, int height,
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
                              float* dL_dcamera, int antialiasing, const float* depth, const float* dL_ddistortion,
                              float* dL_dmean2D_abs) {
    (void)colors_precomp;
    const Api api(__func__);
    if (!depth || !dL_ddistortion) return api.invalid("NULL depth / dL_ddistortion");
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, dL_dmean2D,
                   dL_dconic, dL_dopacity, dL_dcolor, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
                   dL_drot, dL_dz, debug, (cudaStream_t)cuda_stream};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype)) return rc;
    b.dL_dcamera = dL_dcamera;
    b.antialiasing = antialiasing != 0;
    b.depth = depth;
    b.dL_ddistortion = dL_ddistortion;
    b.absgrad = dL_dmean2D_abs != nullptr;
    b.dL_dmean2D_abs = dL_dmean2D_abs;
    return backward(api, b);
}

int f3dgs_backward_accum_distortion(
    int P, int D, int M, int R, int C, const float* background, int width, int height, const float* means3D,
    const float* shs, const float* colors_precomp, const void* semantic_feature, int semantic_feature_dtype,
    const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
    const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
    const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
    const void* dL_dfeaturepix, int dL_dfeaturepix_dtype, float dL_dfeaturepix_scale, const float* dL_depths,
    char* scratch, float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature, float* dL_dmean3D,
    float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dmean2D_out,
    float* grad_accum, float* denom, void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera,
    int antialiasing, const float* depth, const float* dL_ddistortion, float* dL_dmean2D_abs, float* grad_accum_abs) {
    const Api api(__func__);
    if (!depth || !dL_ddistortion) return api.invalid("NULL depth / dL_ddistortion");
    if (grad_accum_abs && !dL_dmean2D_abs) return api.invalid("grad_accum_abs needs dL_dmean2D_abs");
    ViewBackward b{P, D, M, R, C, background, width, height, means3D, shs, scales, scale_modifier, rotations,
                   cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_buffer,
                   binning_buffer, image_buffer, dL_dpix,
                   {dL_dfeaturepix, dL_dfeaturepix_dtype == F3DGS_F16, dL_dfeaturepix_scale}, dL_depths, nullptr,
                   nullptr, dL_dopacity, dL_dcolors_precomp, dL_dsemantic_feature, dL_dmean3D, dL_dcov3D_precomp,
                   dL_dsh, dL_dscale, dL_drot, nullptr, debug, (cudaStream_t)cuda_stream, true, scratch,
                   colors_precomp, dL_dmean2D_out, grad_accum, denom, (cudaEvent_t)composite_done_event};
    if (const int rc = feature_rows(api, b, semantic_feature, semantic_feature_dtype, dL_dfeaturepix_dtype)) return rc;
    b.dL_dcamera = dL_dcamera;
    b.antialiasing = antialiasing != 0;
    b.depth = depth;
    b.dL_ddistortion = dL_ddistortion;
    b.absgrad = dL_dmean2D_abs != nullptr;
    b.dL_dmean2D_abs = dL_dmean2D_abs;
    b.grad_accum_abs = grad_accum_abs;
    return backward(api, b);
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

int f3dgs_gaussian_scores_accum(int P, int R, int width, int height, char* geom_buffer, char* binning_buffer,
                                char* image_buffer, float* weight_sum, float* max_weight, int64_t* pixel_count,
                                void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || R < 0 || width <= 0 || height <= 0)
        return api.invalid("bad sizes (P >= 0, R >= 0, width, height >= 1)");
    if (P == 0 || R == 0) return 0;  // nothing is blended (a forward with R == 0 may leave an empty binning buffer)
    if (!geom_buffer || !binning_buffer || !image_buffer) return api.invalid("missing forward buffers");
    if (!weight_sum || !max_weight || !pixel_count)
        return api.invalid("NULL pointer (weight_sum, max_weight or pixel_count)");
    const Range outs[] = {{weight_sum, (size_t)P * 4}, {max_weight, (size_t)P * 4}, {pixel_count, (size_t)P * 8}};
    for (const Range& r : outs)
        if (overlaps(r, outs)) return api.invalid("weight_sum, max_weight and pixel_count must not overlap");
    const ViewParams vp = make_view(P, 0, 0, 0, width, height, 0.f, 0.f, 1.f, nullptr, nullptr, nullptr);
    return api.cuda(launch_gaussian_scores(vp, forward_buffers(vp, R, geom_buffer, binning_buffer, image_buffer),
                                           weight_sum, max_weight, pixel_count, (cudaStream_t)cuda_stream),
                    "score launch");
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

int f3dgs_densify_plan_absgrad(int P, const float* grad_accum, const float* denom, const float* raw_opacity,
                               const float* raw_scaling, float max_grad, float dense_scale, float min_opacity,
                               float max_world_scale, char* scratch, int32_t* counts, void* cuda_stream,
                               const float* grad_accum_abs, float abs_grad) {
    const Api api(__func__);
    if (P < 0 || 3 * (long long)P > INT_MAX) return api.invalid("bad sizes (0 <= 3 P <= INT_MAX)");
    if (!counts || (P > 0 && (!grad_accum || !denom || !grad_accum_abs || !raw_opacity || !raw_scaling || !scratch)))
        return api.invalid("NULL pointer");
    if (overlaps({counts, 16}, {{scratch, densify_scratch_fixed_bytes(P)}}))
        return api.invalid("counts overlaps scratch");
    return api.cuda(launch_densify_plan(P, grad_accum, denom, raw_opacity, raw_scaling, max_grad, dense_scale,
                                        min_opacity, max_world_scale, scratch, counts, (cudaStream_t)cuda_stream,
                                        grad_accum_abs, abs_grad));
}

int f3dgs_prune_plan(int P, const uint8_t* keep, char* scratch, int32_t* counts, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || 3 * (long long)P > INT_MAX) return api.invalid("bad sizes (0 <= 3 P <= INT_MAX)");
    if (!counts || (P > 0 && (!keep || !scratch))) return api.invalid("NULL pointer");
    const Range flags{scratch, densify_scratch_fixed_bytes(P)};
    if (overlaps(flags, {{keep, (size_t)P}, {counts, 16}})) return api.invalid("keep or counts overlaps scratch");
    return api.cuda(launch_prune_plan(P, keep, scratch, counts, (cudaStream_t)cuda_stream));
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

}  // extern "C"

namespace {
// The 21 pointers of f3dgs_gaussian_fields[3] in order, and their byte ranges over `rows` rows; false if a field of
// nonzero width over rows > 0 is NULL (f_rest has width 0 when M == 1, semantic_feature when C == 0)
bool gaussian_fields(const f3dgs_gaussian_fields f[3], int M, int C, long long rows, float* out[21], Range ranges[21]) {
    const size_t width[7] = {3, 3, 3 * (size_t)(M - 1), 1, 3, 4, (size_t)C};
    for (int g = 0; g < 3; g++) {
        float* p[7] = {f[g].xyz, f[g].f_dc, f[g].f_rest, f[g].opacity, f[g].scaling, f[g].rotation, f[g].semantic_feature};
        for (int j = 0; j < 7; j++) {
            if (width[j] && rows > 0 && !p[j]) return false;
            out[7 * g + j] = p[j];
            ranges[7 * g + j] = {p[j], (size_t)rows * width[j] * 4};
        }
    }
    return true;
}

// Does any of the first `n_out` ranges (the written ones) overlap any other range?
template <size_t N>
bool any_overlap(const Range (&r)[N], size_t n_out) {
    for (size_t i = 0; i < n_out; i++)
        if (overlaps(r[i], r)) return true;
    return false;
}

bool mcmc_sizes_ok(int P, int M, int C) {
    return P >= 0 && 3 * (long long)P <= INT_MAX && M >= 1 && C >= 0 && C <= F3DGS_MAX_FEATURE_DIM;
}
constexpr const char* kMcmcBadSizes = "bad sizes (0 <= 3 P <= INT_MAX, M >= 1, 0 <= C <= F3DGS_MAX_FEATURE_DIM, 0 <= n <= P)";
}  // namespace

extern "C" {

size_t f3dgs_mcmc_scratch_bytes(int P) {
    return scratch_bytes(__func__, [=](size_t* b) { return mcmc_scratch_bytes(P, b); });
}

int f3dgs_mcmc_plan(int P, const float* raw_opacity, float min_opacity, char* scratch, int32_t* n_dead, int32_t* index,
                    float* alive_opacity, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || 3 * (long long)P > INT_MAX) return api.invalid("bad sizes (0 <= 3 P <= INT_MAX)");
    if (!std::isfinite(min_opacity)) return api.invalid("min_opacity must be finite");
    if (!n_dead || (P > 0 && (!raw_opacity || !scratch || !index || !alive_opacity))) return api.invalid("NULL pointer");
    const size_t b = (size_t)P * 4;
    const Range r[5] = {{n_dead, 4}, {index, b}, {alive_opacity, b}, {scratch, mcmc_scratch_fixed_bytes(P)},
                        {raw_opacity, b}};
    if (any_overlap(r, 4)) return api.invalid("n_dead, index, alive_opacity, scratch and raw_opacity overlap");
    return api.cuda(launch_mcmc_plan(P, raw_opacity, min_opacity, scratch, n_dead, index, alive_opacity,
                                     (cudaStream_t)cuda_stream));
}

int f3dgs_mcmc_relocate(int P, int M, int C, int n, const int32_t* dead, const int32_t* src, float min_opacity,
                        const f3dgs_gaussian_fields fields[3], uint16_t* semantic_feature_f16, char* scratch,
                        void* cuda_stream) {
    const Api api(__func__);
    if (!mcmc_sizes_ok(P, M, C) || n < 0 || n > P) return api.invalid(kMcmcBadSizes);
    if (!std::isfinite(min_opacity)) return api.invalid("min_opacity must be finite");
    if (!fields) return api.invalid("NULL pointer");
    Range r[25];
    float* f[21];
    if (!gaussian_fields(fields, M, C, P, f, r)) return api.invalid("NULL pointer (a field)");
    if (n > 0 && (!dead || !src || !scratch)) return api.invalid("NULL pointer");
    r[21] = {semantic_feature_f16, (size_t)P * C * 2};
    r[22] = {scratch, mcmc_scratch_fixed_bytes(P)};
    r[23] = {dead, (size_t)n * 4};
    r[24] = {src, (size_t)n * 4};
    if (any_overlap(r, 23)) return api.invalid("fields, semantic_feature_f16, scratch, dead and src overlap");
    return api.cuda(launch_mcmc_relocate(P, M, C, n, dead, src, min_opacity, f,
                                         reinterpret_cast<__half*>(semantic_feature_f16), scratch,
                                         (cudaStream_t)cuda_stream));
}

int f3dgs_mcmc_add(int P, int M, int C, int n, const int32_t* src, float min_opacity,
                   const f3dgs_gaussian_fields src_fields[3], const f3dgs_gaussian_fields dst_fields[3], char* scratch,
                   void* cuda_stream) {
    const Api api(__func__);
    if (!mcmc_sizes_ok(P, M, C) || n < 0 || n > P || 3 * ((long long)P + n) > INT_MAX) return api.invalid(kMcmcBadSizes);
    if (!std::isfinite(min_opacity)) return api.invalid("min_opacity must be finite");
    if (!src_fields || !dst_fields) return api.invalid("NULL pointer");
    Range r[44];
    float *s[21], *d[21];
    if (!gaussian_fields(dst_fields, M, C, (long long)P + n, d, r) || !gaussian_fields(src_fields, M, C, P, s, r + 21))
        return api.invalid("NULL pointer (a field)");
    if (P > 0 && !scratch) return api.invalid("NULL pointer");
    if (n > 0 && !src) return api.invalid("NULL pointer");
    r[42] = {scratch, mcmc_scratch_fixed_bytes(P)};
    r[43] = {src, (size_t)n * 4};
    // the dst fields and the scratch are written; the src fields may share nothing with them
    bool bad = false;
    for (int i = 0; i < 21 && !bad; i++) bad = overlaps(r[i], r);
    if (bad || overlaps(r[42], r)) return api.invalid("a dst field or the scratch overlaps a field, src or the scratch");
    return api.cuda(launch_mcmc_add(P, M, C, n, src, min_opacity, s, d, scratch, (cudaStream_t)cuda_stream));
}

int f3dgs_mcmc_inject_noise(int P, float* xyz, const float* raw_opacity, const float* raw_scaling,
                            const float* raw_rotation, const float* eps, float scale, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || 4 * (long long)P > INT_MAX) return api.invalid("bad sizes (0 <= 4 P <= INT_MAX)");
    if (!std::isfinite(scale)) return api.invalid("scale must be finite");
    if (P == 0) return 0;
    if (!xyz || !raw_opacity || !raw_scaling || !raw_rotation || !eps) return api.invalid("NULL pointer");
    const size_t b = (size_t)P * 4;
    const Range r[5] = {{xyz, 3 * b}, {raw_opacity, b}, {raw_scaling, 3 * b}, {raw_rotation, 4 * b}, {eps, 3 * b}};
    if (any_overlap(r, 1)) return api.invalid("xyz overlaps raw_opacity, raw_scaling, raw_rotation or eps");
    return api.cuda(launch_mcmc_inject_noise(P, xyz, raw_opacity, raw_scaling, raw_rotation, eps, scale,
                                             (cudaStream_t)cuda_stream));
}

size_t f3dgs_filter3d_scratch_bytes(int P) { return P > 0 ? kFilter3dScratchBytes : 0; }

int f3dgs_filter3d_compute(int P, int V, const float* means3D, const float* viewmatrices, const float* intrinsics,
                           float* filter, int32_t* n_seen, char* scratch, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || 3 * (long long)P > INT_MAX || V < 1 || 16 * (long long)V > INT_MAX)
        return api.invalid("bad sizes (0 <= 3 P <= INT_MAX, 1 <= 16 V <= INT_MAX)");
    if (P == 0) return 0;
    if (!means3D || !viewmatrices || !intrinsics || !filter || !n_seen || !scratch) return api.invalid("NULL pointer");
    const size_t b = (size_t)P * 4;
    const Range r[6] = {{filter, b}, {n_seen, 4}, {scratch, kFilter3dScratchBytes}, {means3D, 3 * b},
                        {viewmatrices, (size_t)V * 64}, {intrinsics, (size_t)V * 16}};
    if (any_overlap(r, 3)) return api.invalid("filter, n_seen, scratch and the inputs overlap");
    return api.cuda(launch_filter3d_compute(P, V, means3D, viewmatrices, intrinsics, filter, n_seen, scratch,
                                            (cudaStream_t)cuda_stream));
}

int f3dgs_filter3d_apply(int P, const float* opacity, const float* scales, const float* filter, float* opacity_out,
                         float* scales_out, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || 3 * (long long)P > INT_MAX) return api.invalid("bad sizes (0 <= 3 P <= INT_MAX)");
    if (P == 0) return 0;
    if (!opacity || !scales || !filter || !opacity_out || !scales_out) return api.invalid("NULL pointer");
    const size_t b = (size_t)P * 4;
    const Range r[5] = {{opacity_out, b}, {scales_out, 3 * b}, {opacity, b}, {scales, 3 * b}, {filter, b}};
    if (any_overlap(r, 2)) return api.invalid("opacity_out, scales_out and the inputs overlap");
    return api.cuda(launch_filter3d_apply(P, opacity, scales, filter, opacity_out, scales_out,
                                          (cudaStream_t)cuda_stream));
}

int f3dgs_filter3d_apply_backward(int P, const float* opacity, const float* scales, const float* filter,
                                  const float* dL_dopacity_f, const float* dL_dscales_f, float* dL_dopacity,
                                  float* dL_dscales, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || 3 * (long long)P > INT_MAX) return api.invalid("bad sizes (0 <= 3 P <= INT_MAX)");
    if (P == 0) return 0;
    if (!opacity || !scales || !filter || !dL_dopacity_f || !dL_dscales_f || !dL_dopacity || !dL_dscales)
        return api.invalid("NULL pointer");
    const size_t b = (size_t)P * 4;
    // an output that is exactly its own upstream gradient is computed in place: that input's range is then the output's
    const Range r[7] = {{dL_dopacity, b}, {dL_dscales, 3 * b}, {opacity, b}, {scales, 3 * b}, {filter, b},
                        {dL_dopacity_f == dL_dopacity ? nullptr : dL_dopacity_f, b},
                        {dL_dscales_f == dL_dscales ? nullptr : dL_dscales_f, 3 * b}};
    if (any_overlap(r, 2)) return api.invalid("an output overlaps an input or the other output (other than in place)");
    return api.cuda(launch_filter3d_apply_backward(P, opacity, scales, filter, dL_dopacity_f, dL_dscales_f, dL_dopacity,
                                                   dL_dscales, (cudaStream_t)cuda_stream));
}

int f3dgs_reset_opacity_filter3d(int P, float* raw_opacity, const float* raw_scaling, const float* filter,
                                 float* exp_avg, float* exp_avg_sq, float ceiling, void* cuda_stream) {
    const Api api(__func__);
    if (P < 0 || 3 * (long long)P > INT_MAX) return api.invalid("bad sizes (0 <= 3 P <= INT_MAX)");
    if (P == 0) return 0;
    if (!raw_opacity || !raw_scaling || !filter || !exp_avg || !exp_avg_sq) return api.invalid("NULL pointer");
    const size_t b = (size_t)P * 4;
    const Range r[5] = {{raw_opacity, b}, {exp_avg, b}, {exp_avg_sq, b}, {raw_scaling, 3 * b}, {filter, b}};
    if (any_overlap(r, 3)) return api.invalid("raw_opacity, exp_avg, exp_avg_sq and the inputs overlap");
    return api.cuda(launch_reset_opacity_filter3d(P, raw_opacity, raw_scaling, filter, exp_avg, exp_avg_sq, ceiling,
                                                  (cudaStream_t)cuda_stream));
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

}  // extern "C"

namespace {
// The checks shared by the masked Adam entries: < 0 the rejection, 0 nothing to do (n == 0), 1 launch
int check_adam_masked(const Api& api, int kind, size_t n, int P, int M, int step, bool null_pointer) {
    if (kind < F3DGS_PARAM_IDENTITY || kind > F3DGS_PARAM_SH_REST) return api.invalid("unknown parameter kind");
    if (step < 0) return api.invalid("step < 0");
    if ((kind == F3DGS_PARAM_SH_DC || kind == F3DGS_PARAM_SH_REST) && M < (kind == F3DGS_PARAM_SH_REST ? 2 : 1))
        return api.invalid("M < 1 for F3DGS_PARAM_SH_DC or M < 2 for F3DGS_PARAM_SH_REST");
    if (n == 0) return 0;
    if (null_pointer) return api.invalid("NULL pointer");
    if (P < 1 || n % (size_t)P != 0) return api.invalid("P < 1 or n % P != 0");
    const size_t width = n / (size_t)P;
    const size_t row[6] = {width, 1, 3, 4, 3, 3 * (size_t)(M - 1)};  // by kind; IDENTITY rows have any width
    if (width != row[kind])
        return api.invalid("n / P is not the row width of the kind (SIGMOID 1, EXP 3, NORMALIZE4 4, SH_DC 3, SH_REST "
                           "3 (M - 1))");
    return 1;
}
}  // namespace

extern "C" {

int f3dgs_adam_step_masked(int kind, size_t n, int P, int M, float* param, const float* grad_activated, float* exp_avg,
                           float* exp_avg_sq, const uint8_t* visible, float lr, float beta1, float beta2, float eps,
                           int step, void* cuda_stream) {
    const Api api(__func__);
    const int rc =
        check_adam_masked(api, kind, n, P, M, step, !param || !grad_activated || !exp_avg || !exp_avg_sq || !visible);
    if (rc <= 0) return rc;
    return api.cuda(launch_adam_step(kind, n, M, param, grad_activated, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, step,
                                     (cudaStream_t)cuda_stream, nullptr, visible, P));
}

int f3dgs_adam_step_masked_f16out(int kind, size_t n, int P, int M, float* param, const float* grad_activated,
                                  float* exp_avg, float* exp_avg_sq, const uint8_t* visible, uint16_t* param_f16,
                                  float lr, float beta1, float beta2, float eps, int step, void* cuda_stream) {
    const Api api(__func__);
    if (kind != F3DGS_PARAM_IDENTITY) return api.invalid("kind must be F3DGS_PARAM_IDENTITY");
    const int rc = check_adam_masked(api, kind, n, P, M, step,
                                     !param || !grad_activated || !exp_avg || !exp_avg_sq || !visible || !param_f16);
    if (rc <= 0) return rc;
    if (overlaps({param_f16, n * 2},
                 {{param, n * 4}, {grad_activated, n * 4}, {exp_avg, n * 4}, {exp_avg_sq, n * 4}, {visible, (size_t)P}}))
        return api.invalid("param_f16 overlaps param, grad_activated, exp_avg, exp_avg_sq or visible");
    return api.cuda(launch_adam_step(kind, n, M, param, grad_activated, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, step,
                                     (cudaStream_t)cuda_stream, reinterpret_cast<__half*>(param_f16), visible, P));
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

namespace {
bool vq_sizes_ok(int P, int K, int D) { return P >= 0 && K >= 1 && K <= kVqMaxK && D >= 1 && D <= kVqMaxD; }
constexpr const char* kVqBadSizes = "bad sizes (P >= 0, 1 <= K <= 65536, 1 <= D <= 4096)";

// the checks shared by update and codebook_grad: < 0 the rejection, 0 nothing to do (P == 0), 1 launch
int check_vq_reduce(const Api& api, int P, int K, int D, const float* x, const float* weights, const char* scratch,
                    const float* out) {
    if (!vq_sizes_ok(P, K, D)) return api.invalid(kVqBadSizes);
    if (P == 0) return 0;
    if (!x || !scratch || !out) return api.invalid("NULL pointer");
    const size_t row = (size_t)D * 4;
    const Range r[4] = {{out, (size_t)K * row}, {x, (size_t)P * row}, {weights, (size_t)P * 4},
                        {scratch, vq_scratch_fixed_bytes(P, K)}};
    if (any_overlap(r, 1)) return api.invalid("the output overlaps x, weights or the scratch");
    return 1;
}

template <typename T>
int vq_decode_impl(const char* entry, int P, int K, int D, const float* codebook, const int32_t* code, T* out,
                   void* cuda_stream) {
    const Api api(entry);
    if (!vq_sizes_ok(P, K, D)) return api.invalid(kVqBadSizes);
    if (P == 0) return 0;
    if (!codebook || !code || !out) return api.invalid("NULL pointer");
    const Range r[3] = {{out, (size_t)P * D * sizeof(T)}, {codebook, (size_t)K * D * 4}, {code, (size_t)P * 4}};
    if (any_overlap(r, 1)) return api.invalid("out overlaps the codebook or code");
    return api.cuda(launch_vq_decode(P, K, D, codebook, code, out, (cudaStream_t)cuda_stream));
}
}  // namespace

extern "C" {

size_t f3dgs_vq_scratch_bytes(int P, int K) {
    if (K < 1 || K > kVqMaxK) return 0;
    return scratch_bytes(__func__, [=](size_t* b) { return vq_scratch_bytes(P, K, b); });
}

int f3dgs_vq_assign(int P, int K, int D, const float* x, const float* codebook, int32_t* code, void* cuda_stream) {
    const Api api(__func__);
    if (!vq_sizes_ok(P, K, D)) return api.invalid(kVqBadSizes);
    if (P == 0) return 0;
    if (!x || !codebook || !code) return api.invalid("NULL pointer");
    const Range r[3] = {{code, (size_t)P * 4}, {x, (size_t)P * D * 4}, {codebook, (size_t)K * D * 4}};
    if (any_overlap(r, 1)) return api.invalid("code overlaps x or the codebook");
    return api.cuda(launch_vq_assign(P, K, D, x, codebook, code, (cudaStream_t)cuda_stream));
}

int f3dgs_vq_plan(int P, int K, const int32_t* code, char* scratch, void* cuda_stream) {
    const Api api(__func__);
    if (!vq_sizes_ok(P, K, 1)) return api.invalid(kVqBadSizes);
    if (P == 0) return 0;
    if (!code || !scratch) return api.invalid("NULL pointer");
    const Range r[2] = {{scratch, vq_scratch_fixed_bytes(P, K)}, {code, (size_t)P * 4}};
    if (any_overlap(r, 1)) return api.invalid("scratch overlaps code");
    size_t sb = 0;
    CUDA_TRY(vq_scratch_bytes(P, K, &sb));  // the sort's share of the scratch is sized by CUB for the current device
    if (overlaps({code, (size_t)P * 4}, {{scratch, sb}})) return api.invalid("scratch overlaps code");
    return api.cuda(launch_vq_plan(P, K, code, scratch, (cudaStream_t)cuda_stream));
}

int f3dgs_vq_update(int P, int K, int D, const float* x, const float* weights, const char* scratch, float* codebook,
                    void* cuda_stream) {
    const Api api(__func__);
    const int rc = check_vq_reduce(api, P, K, D, x, weights, scratch, codebook);
    if (rc <= 0) return rc;
    return api.cuda(launch_vq_reduce(P, K, D, x, weights, scratch, codebook, true, (cudaStream_t)cuda_stream));
}

int f3dgs_vq_codebook_grad(int P, int K, int D, const float* dL_dx, const char* scratch, float* dL_dcodebook,
                           void* cuda_stream) {
    const Api api(__func__);
    const int rc = check_vq_reduce(api, P, K, D, dL_dx, nullptr, scratch, dL_dcodebook);
    if (rc <= 0) return rc;
    return api.cuda(launch_vq_reduce(P, K, D, dL_dx, nullptr, scratch, dL_dcodebook, false, (cudaStream_t)cuda_stream));
}

int f3dgs_vq_decode(int P, int K, int D, const float* codebook, const int32_t* code, float* out, void* cuda_stream) {
    return vq_decode_impl(__func__, P, K, D, codebook, code, out, cuda_stream);
}

int f3dgs_vq_decode_f16out(int P, int K, int D, const float* codebook, const int32_t* code, uint16_t* out,
                           void* cuda_stream) {
    return vq_decode_impl(__func__, P, K, D, codebook, code, reinterpret_cast<__half*>(out), cuda_stream);
}

}  // extern "C"

namespace {
bool knn_graph_sizes_ok(int P, int k) { return P >= 0 && k >= 1 && k <= 32 && (long long)P * k <= INT_MAX; }
constexpr const char* kKnnGraphBadSizes = "bad sizes (P >= 0, 1 <= k <= 32, P k <= 2^31 - 1)";
}  // namespace

extern "C" {

size_t f3dgs_knn_graph_scratch_bytes(int P, int k) {
    if (!knn_graph_sizes_ok(P, k)) return 0;
    return scratch_bytes(__func__, [=](size_t* b) { return knn_graph_scratch_bytes(P, k, b); });
}

int f3dgs_knn_graph(int P, int k, const float* points, int32_t* idx, float* dist2, int32_t* order, char* scratch,
                    void* cuda_stream) {
    const Api api(__func__);
    if (!knn_graph_sizes_ok(P, k)) return api.invalid(kKnnGraphBadSizes);
    if (P == 0) return 0;
    if (!points || !idx || !dist2 || !order || !scratch) return api.invalid("NULL pointer");
    const size_t E = (size_t)P * k;
    Range r[5] = {{idx, E * 4}, {dist2, E * 4}, {order, (size_t)P * 4}, {points, (size_t)P * 12},
                  {scratch, knn_graph_scratch_fixed_bytes(P, k)}};
    if (any_overlap(r, 3)) return api.invalid("idx, dist2 and order overlap each other, points or scratch");
    size_t sb = 0;
    CUDA_TRY(knn_graph_scratch_bytes(P, k, &sb));  // the sorts' share of the scratch is sized by CUB for the device
    r[4].bytes = sb;
    if (any_overlap(r, 3)) return api.invalid("idx, dist2 and order overlap each other, points or scratch");
    return api.cuda(launch_knn_graph(P, k, points, idx, dist2, order, scratch, (cudaStream_t)cuda_stream));
}

int f3dgs_knn_reverse(int P, int k, const int32_t* idx, int32_t* offsets, int32_t* sources, char* scratch,
                      void* cuda_stream) {
    const Api api(__func__);
    if (!knn_graph_sizes_ok(P, k)) return api.invalid(kKnnGraphBadSizes);
    if (P == 0) return 0;
    if (!idx || !offsets || !sources || !scratch) return api.invalid("NULL pointer");
    const size_t E = (size_t)P * k;
    Range r[4] = {{offsets, ((size_t)P + 1) * 4}, {sources, E * 4}, {idx, E * 4},
                  {scratch, knn_graph_scratch_fixed_bytes(P, k)}};
    if (any_overlap(r, 2)) return api.invalid("offsets and sources overlap each other, idx or scratch");
    size_t sb = 0;
    CUDA_TRY(knn_graph_scratch_bytes(P, k, &sb));
    r[3].bytes = sb;
    if (any_overlap(r, 2)) return api.invalid("offsets and sources overlap each other, idx or scratch");
    return api.cuda(launch_knn_reverse(P, k, idx, offsets, sources, scratch, (cudaStream_t)cuda_stream));
}

int f3dgs_feature_tv_accum(int P, int k, int C, const float* features, const int32_t* idx, const int32_t* offsets,
                           const int32_t* sources, const int32_t* order, double weight, long long n_edges, float* grad,
                           double* loss, void* cuda_stream) {
    const Api api(__func__);
    if (!knn_graph_sizes_ok(P, k) || C < 1 || C > F3DGS_MAX_FEATURE_DIM || n_edges < 0 || n_edges > (long long)P * k)
        return api.invalid("bad sizes (P >= 0, 1 <= k <= 32, P k <= 2^31 - 1, 1 <= C <= F3DGS_MAX_FEATURE_DIM, "
                           "0 <= n_edges <= P k)");
    if (!std::isfinite(weight)) return api.invalid("weight must be finite");
    if (P == 0) return 0;
    if (!features || !idx || !offsets || !sources || !grad || !loss) return api.invalid("NULL pointer");
    const size_t E = (size_t)P * k, row = (size_t)C * 4;
    const Range r[7] = {{grad, (size_t)P * row}, {loss, 8}, {features, (size_t)P * row}, {idx, E * 4},
                        {offsets, ((size_t)P + 1) * 4}, {sources, E * 4}, {order, (size_t)P * 4}};
    if (any_overlap(r, 2)) return api.invalid("grad and loss overlap each other or an input");
    const cudaError_t e = launch_feature_tv_accum(P, k, C, features, idx, offsets, sources, order, weight, n_edges,
                                                  grad, loss, (cudaStream_t)cuda_stream);
    if (e == cudaErrorMemoryAllocation)
        return api.fail(F3DGS_ERR_ALLOC, std::string("cudaMallocAsync for the partial sums failed: ") +
                                             cudaGetErrorString(e));
    return api.cuda(e);
}

int f3dgs_feature_fill(int P, int k, int C, const float* features, const float* weights, const int32_t* idx,
                       float min_weight, float* out, void* cuda_stream) {
    const Api api(__func__);
    if (!knn_graph_sizes_ok(P, k) || C < 1 || C > F3DGS_MAX_FEATURE_DIM)
        return api.invalid("bad sizes (P >= 0, 1 <= k <= 32, P k <= 2^31 - 1, 1 <= C <= F3DGS_MAX_FEATURE_DIM)");
    if (std::isnan(min_weight)) return api.invalid("min_weight must not be NaN");
    if (P == 0) return 0;
    if (!features || !weights || !idx || !out) return api.invalid("NULL pointer");
    const size_t row = (size_t)C * 4;
    const Range r[4] = {{out, (size_t)P * row}, {features, (size_t)P * row}, {weights, (size_t)P * 4},
                        {idx, (size_t)P * k * 4}};
    if (any_overlap(r, 1)) return api.invalid("out overlaps features, weights or idx");
    return api.cuda(launch_feature_fill(P, k, C, features, weights, idx, min_weight, out, (cudaStream_t)cuda_stream));
}

}  // extern "C"
