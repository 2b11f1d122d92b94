// torch / pybind11 surface `diff_gaussian_rasterization._C` over the C ABI of libf3dgs_b200.so.
//
// Same three functions, positional signatures and return tuples as the reference module
// (reference ext.cpp:15-19, rasterize_points.h:18-72, rasterize_points.cu:35-236), so the
// reference's Python wrapper logic calls it unchanged:
//   rasterize_gaussians(...)          -> (num_rendered, color, feature_map, depth, radii, geom, binning, img)
//   rasterize_gaussians_backward(...) -> (dL_dmeans2D, dL_dcolors, dL_dsemantic_feature, dL_dopacity,
//                                         dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations)
//   mark_visible(means3D, viewmatrix, projmatrix) -> bool[P]
// plus rasterize_gaussians_backward_camera(same arguments as rasterize_gaussians_backward) -> its 9 gradients +
// (dL_dviewmatrix [4,4], dL_dprojmatrix [4,4], dL_dcampos [3]) for pose refinement (f3dgs_backward_cam), and
// rasterize_gaussians_backward_feature_geometry(same arguments, camera) -> the same 12 (the camera three None unless
// `camera`) with the feature term of dL/dalpha (f3dgs_backward_feature_geometry).  Antialiased rendering:
// rasterize_gaussians_antialiased (rasterize_gaussians' arguments and results, f3dgs_forward_antialiased) and
// rasterize_gaussians_backward_antialiased(same arguments, camera=False, semantic_feature=None) -> the same 12, with the
// feature term when semantic_feature is given (f3dgs_backward_antialiased).  Opacity and inverse-depth maps:
// rasterize_gaussians_alpha_invdepth(rasterize_gaussians' arguments, antialiasing=False) -> (num_rendered, color,
// feature_map, depth, alpha, invdepth, radii, geom, binning, img) (f3dgs_forward_alpha_invdepth) and
// rasterize_gaussians_backward_alpha_invdepth(the backward's arguments, dL_dout_alpha, dL_dout_invdepth, camera=False,
// semantic_feature=None, antialiasing=False) -> the same 12 as rasterize_gaussians_backward_antialiased
// (f3dgs_backward_alpha_invdepth).
// Differences (all permissive): the feature width is read from semantic_feature.size(-1) at run
// time (reference: compile-time NUM_SEMANTIC_CHANNELS, config.h:16); an empty / undefined
// semantic_feature means C = 0; semantic_feature may be float32 or float16, and the feature map
// has its dtype (f3dgs_forward / f3dgs_forward_f16); the backward calls take a float32 or float16 feature-map
// gradient (f3dgs_backward_f16 / f3dgs_backward_accum_f16); inputs are checked for device/dtype and errors
// from the C ABI are raised as RuntimeError.  This file contains no CUDA code and there is no CPU
// fallback.
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/extension.h>

#include <string>
#include <tuple>
#include <vector>

#include "../../include/f3dgs_b200.h"

namespace {

// reference rasterize_points.cu:27-33 (resizeFunctional): grow a uint8 CUDA tensor on demand
char* resize_tensor(void* ctx, size_t bytes) {
    auto* t = static_cast<torch::Tensor*>(ctx);
    t->resize_({(long long)bytes});
    return reinterpret_cast<char*>(t->data_ptr());
}

const float* fptr(const torch::Tensor& t) {  // empty tensor -> nullptr, as in the reference
    if (!t.defined() || t.numel() == 0) return nullptr;
    return t.data_ptr<float>();
}

// The two tensor checks.  An undefined or empty tensor is an absent argument for both.
// A float32 input on `dev` that is only read: made contiguous (a copy if it is not).
torch::Tensor input(const torch::Tensor& t, const torch::Device& dev, const char* name) {
    if (!t.defined() || t.numel() == 0) return t;
    TORCH_CHECK(t.scalar_type() == torch::kFloat32, name, " must be float32");
    TORCH_CHECK(t.device() == dev, name, " must be on ", dev, " (got ", t.device(), ")");
    return t.contiguous();
}
// A float32 tensor of `numel` elements on `dev` that the call reads or writes in place, so it must be contiguous already
// -> its data, or nullptr if absent.
float* in_place(const torch::Tensor& t, const torch::Device& dev, int64_t numel, const char* name) {
    if (!t.defined() || t.numel() == 0) return nullptr;
    TORCH_CHECK(t.is_cuda() && t.device() == dev && t.scalar_type() == torch::kFloat32 && t.is_contiguous() &&
                    t.numel() == numel,
                name, " must be a contiguous float32 tensor of ", numel, " elements on ", dev, " (got ", t.numel(),
                " elements of ", t.scalar_type(), " on ", t.device(), ")");
    return t.data_ptr<float>();
}

// semantic_feature of the rasterizer calls: float32 or float16 on `dev` (the feature map takes its dtype); undefined or
// empty is absent, as for input()
void check_features(const torch::Tensor& t, const torch::Device& dev) {
    if (!t.defined() || t.numel() == 0) return;
    TORCH_CHECK(t.scalar_type() == torch::kFloat32 || t.scalar_type() == torch::kFloat16,
                "semantic_feature must be float32 or float16 (got ", t.scalar_type(), ")");
    TORCH_CHECK(t.device() == dev, "semantic_feature must be on ", dev, " (got ", t.device(), ")");
}

// dL/dfeature_map of the backward calls: float32 or float16 [C,H,W] on `dev`, made contiguous; undefined or empty is absent
torch::Tensor feature_grad(const torch::Tensor& t, const torch::Device& dev) {
    if (!t.defined() || t.numel() == 0) return t;
    TORCH_CHECK(t.scalar_type() == torch::kFloat32 || t.scalar_type() == torch::kFloat16,
                "grad_out_feature must be float32 or float16 (got ", t.scalar_type(), ")");
    TORCH_CHECK(t.device() == dev, "grad_out_feature must be on ", dev, " (got ", t.device(), ")");
    return t.contiguous();
}

// The gradient of an opacity or inverse-depth plane: float32 [1,H,W] (any shape of H*W elements) on `dev`, made
// contiguous; undefined or empty stands for zeros
torch::Tensor plane_grad(const torch::Tensor& t, const torch::Device& dev, int64_t H, int64_t W, const char* name) {
    if (!t.defined() || t.numel() == 0) return torch::zeros({1, H, W}, torch::TensorOptions().device(dev));
    TORCH_CHECK(t.numel() == H * W, name, " must have H * W = ", H * W, " elements (got ", t.numel(), ")");
    return input(t, dev, name);
}

// C-ABI element-type code of a float32 or float16 tensor (absent: float32)
int dtype_code(const torch::Tensor& t) {
    return t.defined() && t.scalar_type() == torch::kFloat16 ? F3DGS_F16 : F3DGS_F32;
}

void check_rc(int rc, const char* what) {
    TORCH_CHECK(rc >= 0, what, " failed (code ", -rc, "): ", f3dgs_last_error());
}

// Calls the float16 twin of a C-ABI function with t's IEEE binary16 bits if t is float16, else the float32 one with t's
// float data; `call(fn, ptr)` writes the argument list once for both.
template <typename F32, typename F16, typename Call>
void call_f32_or_f16(const torch::Tensor& t, F32 f32, const char* name32, F16 f16, const char* name16, Call call) {
    if (t.defined() && t.scalar_type() == torch::kFloat16)
        check_rc(call(f16, reinterpret_cast<uint16_t*>(t.data_ptr<at::Half>())), name16);
    else
        check_rc(call(f32, const_cast<float*>(fptr(t))), name32);
}

// A scratch tensor of the size a f3dgs_*_scratch_bytes function returned: 0 is a failure when it set the last error
torch::Tensor scratch_tensor(size_t bytes, const char* fn, const torch::Tensor& like) {
    TORCH_CHECK(bytes > 0 || f3dgs_last_error()[0] == '\0', fn, " failed: ", f3dgs_last_error());
    return torch::empty({(int64_t)bytes}, like.options().dtype(torch::kByte));
}

}  // namespace

using ForwardResults = std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
                                  torch::Tensor, torch::Tensor>;

#define FORWARD_PARAMS                                                                                                 \
    const torch::Tensor &background, const torch::Tensor &means3D, const torch::Tensor &colors,                       \
        const torch::Tensor &semantic_feature, const torch::Tensor &opacity, const torch::Tensor &scales,             \
        const torch::Tensor &rotations, const float scale_modifier, const torch::Tensor &cov3D_precomp,               \
        const torch::Tensor &viewmatrix, const torch::Tensor &projmatrix, const float tan_fovx, const float tan_fovy, \
        const int image_height, const int image_width, const torch::Tensor &sh, const int degree,                     \
        const torch::Tensor &campos, const bool prefiltered, const bool debug
#define FORWARD_ARGS                                                                                                   \
    background, means3D, colors, semantic_feature, opacity, scales, rotations, scale_modifier, cov3D_precomp,         \
        viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, debug

// Body of rasterize_gaussians, rasterize_gaussians_antialiased (f3dgs_forward_antialiased) and, with `planes` (two
// tensors it sets to the [1,H,W] opacity and inverse-depth planes), rasterize_gaussians_alpha_invdepth
// (f3dgs_forward_alpha_invdepth)
static ForwardResults forward(FORWARD_PARAMS, const bool antialiasing, torch::Tensor* planes = nullptr) {
    if (means3D.ndimension() != 2 || means3D.size(1) != 3) {
        AT_ERROR("means3D must have dimensions (num_points, 3)");
    }
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor (this build has no CPU path)");
    const c10::cuda::CUDAGuard guard(means3D.device());
    const auto dev = means3D.device();
    const int P = means3D.size(0);
    const int H = image_height, W = image_width;
    // feature width = last dimension (also for an empty cloud [0,1,C]); an absent feature input is a 0-element 1-D tensor
    const int C = (semantic_feature.defined() && semantic_feature.dim() >= 1) ? (int)semantic_feature.size(-1) : 0;
    TORCH_CHECK(!semantic_feature.defined() || semantic_feature.numel() == (int64_t)P * C,
                "semantic_feature must be [P, 1, C]");

    auto float_opts = means3D.options().dtype(torch::kFloat32);
    const bool half = semantic_feature.defined() && semantic_feature.scalar_type() == torch::kFloat16;
    auto feat_opts = means3D.options().dtype(half ? torch::kFloat16 : torch::kFloat32);
    // every element of the outputs is written by the composite kernel, so no zero-fill pass
    // (reference: torch::full 0, rasterize_points.cu:67-73); P == 0 keeps the reference's zeros
    torch::Tensor out_color = P ? torch::empty({3, H, W}, float_opts) : torch::zeros({3, H, W}, float_opts);
    torch::Tensor out_depth = P ? torch::empty({1, H, W}, float_opts) : torch::zeros({1, H, W}, float_opts);
    torch::Tensor out_feature = P ? torch::empty({C, H, W}, feat_opts) : torch::zeros({C, H, W}, feat_opts);
    torch::Tensor radii = torch::empty({P}, means3D.options().dtype(torch::kInt32));
    if (planes)
        for (int k = 0; k < 2; k++) planes[k] = P ? torch::empty({1, H, W}, float_opts) : torch::zeros({1, H, W}, float_opts);

    auto byte_opts = torch::TensorOptions().dtype(torch::kByte).device(dev);
    torch::Tensor geomBuffer = torch::empty({0}, byte_opts);
    torch::Tensor binningBuffer = torch::empty({0}, byte_opts);
    torch::Tensor imgBuffer = torch::empty({0}, byte_opts);

    int rendered = 0;
    if (P != 0) {
        int M = 0;
        if (sh.defined() && sh.numel() != 0) M = sh.size(1);
        check_features(semantic_feature, dev);
        auto bg = input(background, dev, "bg"), m3 = input(means3D, dev, "means3D");
        auto col = input(colors, dev, "colors_precomp");
        const bool has_sf = semantic_feature.defined() && semantic_feature.numel();
        auto sf = has_sf ? semantic_feature.contiguous() : semantic_feature;
        auto op = input(opacity, dev, "opacities"), sc = input(scales, dev, "scales");
        auto rot = input(rotations, dev, "rotations"), cov = input(cov3D_precomp, dev, "cov3D_precomp");
        auto vm = input(viewmatrix, dev, "viewmatrix"), pm = input(projmatrix, dev, "projmatrix");
        auto shc = input(sh, dev, "shs"), cp = input(campos, dev, "campos");
        cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
        if (planes) {
            rendered = f3dgs_forward_alpha_invdepth(
                resize_tensor, &geomBuffer, resize_tensor, &binningBuffer, resize_tensor, &imgBuffer, P, degree, M, C,
                fptr(bg), W, H, fptr(m3), fptr(shc), fptr(col), has_sf ? sf.data_ptr() : nullptr, dtype_code(sf),
                fptr(op), fptr(sc), scale_modifier, fptr(rot), fptr(cov), fptr(vm), fptr(pm), fptr(cp), tan_fovx,
                tan_fovy, prefiltered ? 1 : 0, out_color.data_ptr<float>(), C ? out_feature.data_ptr() : nullptr,
                out_depth.data_ptr<float>(), radii.data_ptr<int>(), debug ? 1 : 0, (void*)stream, antialiasing ? 1 : 0,
                planes[0].data_ptr<float>(), planes[1].data_ptr<float>());
            check_rc(rendered, "f3dgs_forward_alpha_invdepth");
        } else if (antialiasing) {
            rendered = f3dgs_forward_antialiased(
                resize_tensor, &geomBuffer, resize_tensor, &binningBuffer, resize_tensor, &imgBuffer, P, degree, M, C,
                fptr(bg), W, H, fptr(m3), fptr(shc), fptr(col), has_sf ? sf.data_ptr() : nullptr, dtype_code(sf),
                fptr(op), fptr(sc), scale_modifier, fptr(rot), fptr(cov), fptr(vm), fptr(pm), fptr(cp), tan_fovx,
                tan_fovy, prefiltered ? 1 : 0, out_color.data_ptr<float>(), C ? out_feature.data_ptr() : nullptr,
                out_depth.data_ptr<float>(), radii.data_ptr<int>(), debug ? 1 : 0, (void*)stream);
            check_rc(rendered, "f3dgs_forward_antialiased");
        } else
        call_f32_or_f16(sf, f3dgs_forward, "f3dgs_forward", f3dgs_forward_f16, "f3dgs_forward_f16",
                        [&](auto fn, auto sp) {  // sp: float* or uint16_t*, and the feature map is of the same type
                            auto* fm = C ? static_cast<decltype(sp)>(out_feature.data_ptr()) : nullptr;
                            return rendered = fn(resize_tensor, &geomBuffer, resize_tensor, &binningBuffer,
                                                 resize_tensor, &imgBuffer, P, degree, M, C, fptr(bg), W, H, fptr(m3),
                                                 fptr(shc), fptr(col), sp, fptr(op), fptr(sc), scale_modifier,
                                                 fptr(rot), fptr(cov), fptr(vm), fptr(pm), fptr(cp), tan_fovx,
                                                 tan_fovy, prefiltered ? 1 : 0, out_color.data_ptr<float>(), fm,
                                                 out_depth.data_ptr<float>(), radii.data_ptr<int>(), debug ? 1 : 0,
                                                 (void*)stream);
                        });
    }
    return std::make_tuple(rendered, out_color, out_feature, out_depth, radii, geomBuffer, binningBuffer, imgBuffer);
}

ForwardResults RasterizeGaussiansCUDA(FORWARD_PARAMS) { return forward(FORWARD_ARGS, false); }
ForwardResults RasterizeGaussiansAntialiasedCUDA(FORWARD_PARAMS) { return forward(FORWARD_ARGS, true); }
std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
           torch::Tensor, torch::Tensor>
RasterizeGaussiansAlphaInvDepthCUDA(FORWARD_PARAMS, const bool antialiasing) {
    torch::Tensor planes[2];
    const auto [rendered, color, feature, depth, radii, geom, binning, img] = forward(FORWARD_ARGS, antialiasing, planes);
    return std::make_tuple(rendered, color, feature, depth, planes[0], planes[1], radii, geom, binning, img);
}
#undef FORWARD_PARAMS
#undef FORWARD_ARGS

using BackwardGrads = std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
                                 torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;

// Body of rasterize_gaussians_backward, _camera, _feature_geometry and _antialiased: with a non-NULL camera (35 floats on
// the device), the _cam entries, which add the camera gradient to it; with feature_geometry,
// f3dgs_backward_feature_geometry, which reads semantic_feature and takes the camera gradient as an optional argument;
// with antialiasing, f3dgs_backward_antialiased, whose feature term reads `features` if that is given; with `planes`
// (the gradients of the opacity and inverse-depth planes), f3dgs_backward_alpha_invdepth, with the feature term as under
// antialiasing and the forward's mode `antialiasing`
static BackwardGrads backward_grads(const torch::Tensor& background, const torch::Tensor& means3D,
                               const torch::Tensor& radii, const torch::Tensor& colors,
                               const torch::Tensor& semantic_feature, const torch::Tensor& scales,
                               const torch::Tensor& rotations, const float scale_modifier,
                               const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                               const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                               const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_feature,
                               const torch::Tensor& dL_dout_depth, const torch::Tensor& sh, const int degree,
                               const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R,
                               const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer,
                               const bool debug, float* camera, bool feature_geometry = false,
                               bool antialiasing = false, const torch::Tensor& features = torch::Tensor(),
                               const torch::Tensor* planes = nullptr) {
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor (this build has no CPU path)");
    const c10::cuda::CUDAGuard guard(means3D.device());
    const auto dev = means3D.device();
    const int P = means3D.size(0);
    const int H = dL_dout_color.size(1);
    const int W = dL_dout_color.size(2);
    int M = 0;
    if (sh.defined() && sh.numel() != 0) M = sh.size(1);
    const int C = (semantic_feature.defined() && semantic_feature.dim() >= 1) ? (int)semantic_feature.size(-1) : 0;
    const int64_t mid = (semantic_feature.defined() && semantic_feature.dim() == 3) ? semantic_feature.size(1) : 1;

    auto o = means3D.options().dtype(torch::kFloat32);
    torch::Tensor dL_dmeans3D = torch::zeros({P, 3}, o);
    torch::Tensor dL_dmeans2D = torch::zeros({P, 3}, o);
    torch::Tensor dL_dcolors = torch::zeros({P, 3}, o);
    torch::Tensor dL_dsemantic_feature = torch::zeros({P, mid, C}, o);
    torch::Tensor dL_dconic = torch::zeros({P, 2, 2}, o);
    torch::Tensor dL_dopacity = torch::zeros({P, 1}, o);
    torch::Tensor dL_dcov3D = torch::zeros({P, 6}, o);
    torch::Tensor dL_dsh = torch::zeros({P, M, 3}, o);
    torch::Tensor dL_dscales = torch::zeros({P, 3}, o);
    torch::Tensor dL_drotations = torch::zeros({P, 4}, o);
    torch::Tensor dL_dz = torch::zeros({P, 1}, o);

    if (P != 0) {
        // only semantic_feature's shape is used: dL/dfeature depends on the blend weights alone (f3dgs_backward does
        // not read the features), so a float16 one needs no float32 copy
        check_features(semantic_feature, dev);
        auto bg = input(background, dev, "bg"), m3 = input(means3D, dev, "means3D");
        auto col = input(colors, dev, "colors_precomp");
        auto sc = input(scales, dev, "scales"), rot = input(rotations, dev, "rotations");
        auto cov = input(cov3D_precomp, dev, "cov3D_precomp");
        auto vm = input(viewmatrix, dev, "viewmatrix"), pm = input(projmatrix, dev, "projmatrix");
        auto shc = input(sh, dev, "shs"), cp = input(campos, dev, "campos");
        auto gc = input(dL_dout_color, dev, "grad_out_color");
        auto gd = input(dL_dout_depth, dev, "grad_out_depth");
        // a float16 map gradient goes to f3dgs_backward_f16 as it is (scale 1), without a float32 copy
        torch::Tensor gf = C ? feature_grad(dL_dout_feature, dev) : torch::Tensor();
        TORCH_CHECK(radii.scalar_type() == torch::kInt32 && radii.is_cuda(), "radii must be int32 CUDA");
        auto rad = radii.contiguous();
        auto gb = geomBuffer.contiguous(), bb = binningBuffer.contiguous(), ib = imageBuffer.contiguous();
        cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
        // scale: the float16 symbol's scale after the map, () for the float32 one; tail: (dL_dcamera) or ()
        auto run = [&](auto fn, auto gp, auto scale, auto tail) {
            return std::apply(
                fn, std::tuple_cat(
                        std::make_tuple(P, degree, M, R, C, fptr(bg), W, H, fptr(m3), fptr(shc), fptr(col), nullptr,
                                        fptr(sc), scale_modifier, fptr(rot), fptr(cov), fptr(vm), fptr(pm), fptr(cp),
                                        tan_fovx, tan_fovy, rad.data_ptr<int>(), reinterpret_cast<char*>(gb.data_ptr()),
                                        reinterpret_cast<char*>(bb.data_ptr()), reinterpret_cast<char*>(ib.data_ptr()),
                                        fptr(gc), gp),
                        scale,
                        std::make_tuple(fptr(gd), dL_dmeans2D.data_ptr<float>(), dL_dconic.data_ptr<float>(),
                                        dL_dopacity.data_ptr<float>(), dL_dcolors.data_ptr<float>(),
                                        C ? dL_dsemantic_feature.data_ptr<float>() : nullptr,
                                        dL_dmeans3D.data_ptr<float>(), dL_dcov3D.data_ptr<float>(),
                                        M ? dL_dsh.data_ptr<float>() : nullptr, dL_dscales.data_ptr<float>(),
                                        dL_drotations.data_ptr<float>(), dL_dz.data_ptr<float>(), debug ? 1 : 0,
                                        (void*)stream),
                        tail));
        };
        auto dispatch = [&](auto tail) {
            return [&, tail](auto fn, auto gp) {
                if constexpr (std::is_same_v<decltype(gp), uint16_t*>) return run(fn, gp, std::make_tuple(1.0f), tail);
                else return run(fn, gp, std::tuple<>(), tail);
            };
        };
        // the _feature_geometry / _antialiased entries: features sf (its element type by code; NULL if absent or C == 0)
        auto typed_call = [&](auto fn, const torch::Tensor& sf, auto... tail) {
            return fn(P, degree, M, R, C, fptr(bg), W, H, fptr(m3), fptr(shc), fptr(col),
                      C && sf.defined() && sf.numel() ? sf.data_ptr() : nullptr, dtype_code(sf), fptr(sc),
                      scale_modifier, fptr(rot), fptr(cov), fptr(vm), fptr(pm), fptr(cp), tan_fovx, tan_fovy,
                      rad.data_ptr<int>(), reinterpret_cast<char*>(gb.data_ptr()), reinterpret_cast<char*>(bb.data_ptr()),
                      reinterpret_cast<char*>(ib.data_ptr()), fptr(gc), gf.defined() ? gf.data_ptr() : nullptr,
                      dtype_code(gf), 1.0f, fptr(gd), dL_dmeans2D.data_ptr<float>(), dL_dconic.data_ptr<float>(),
                      dL_dopacity.data_ptr<float>(), dL_dcolors.data_ptr<float>(),
                      C ? dL_dsemantic_feature.data_ptr<float>() : nullptr, dL_dmeans3D.data_ptr<float>(),
                      dL_dcov3D.data_ptr<float>(), M ? dL_dsh.data_ptr<float>() : nullptr, dL_dscales.data_ptr<float>(),
                      dL_drotations.data_ptr<float>(), dL_dz.data_ptr<float>(), debug ? 1 : 0, (void*)stream, camera,
                      tail...);
        };
        // these entries read the features themselves, not only their shape
        auto feature_rows = [&](const torch::Tensor& t) {
            if (!t.defined() || t.numel() == 0) return t;
            check_features(t, dev);
            TORCH_CHECK(!C || t.numel() == (int64_t)P * C, "semantic_feature must have P * C = ", (int64_t)P * C,
                        " elements (got ", t.numel(), ")");
            return t.contiguous();
        };
        if (planes) {
            auto ga = plane_grad(planes[0], dev, H, W, "dL_dout_alpha"), gi = plane_grad(planes[1], dev, H, W,
                                                                                       "dL_dout_invdepth");
            check_rc(typed_call(f3dgs_backward_alpha_invdepth, feature_rows(features), antialiasing ? 1 : 0, fptr(ga),
                                fptr(gi)),
                     "f3dgs_backward_alpha_invdepth");
        } else if (antialiasing)
            check_rc(typed_call(f3dgs_backward_antialiased, feature_rows(features)), "f3dgs_backward_antialiased");
        else if (feature_geometry)
            check_rc(typed_call(f3dgs_backward_feature_geometry, feature_rows(semantic_feature)),
                     "f3dgs_backward_feature_geometry");
        else if (camera)
            call_f32_or_f16(gf, f3dgs_backward_cam, "f3dgs_backward_cam", f3dgs_backward_cam_f16,
                            "f3dgs_backward_cam_f16", dispatch(std::make_tuple(camera)));
        else
            call_f32_or_f16(gf, f3dgs_backward, "f3dgs_backward", f3dgs_backward_f16, "f3dgs_backward_f16",
                            dispatch(std::tuple<>()));
    }
    return std::make_tuple(dL_dmeans2D, dL_dcolors, dL_dsemantic_feature, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh,
                           dL_dscales, dL_drotations);
}

#define BACKWARD_PARAMS                                                                                                \
    const torch::Tensor &background, const torch::Tensor &means3D, const torch::Tensor &radii,                        \
        const torch::Tensor &colors, const torch::Tensor &semantic_feature, const torch::Tensor &scales,              \
        const torch::Tensor &rotations, const float scale_modifier, const torch::Tensor &cov3D_precomp,               \
        const torch::Tensor &viewmatrix, const torch::Tensor &projmatrix, const float tan_fovx, const float tan_fovy, \
        const torch::Tensor &dL_dout_color, const torch::Tensor &dL_dout_feature, const torch::Tensor &dL_dout_depth, \
        const torch::Tensor &sh, const int degree, const torch::Tensor &campos, const torch::Tensor &geomBuffer,       \
        const int R, const torch::Tensor &binningBuffer, const torch::Tensor &imageBuffer, const bool debug
#define BACKWARD_ARGS                                                                                                  \
    background, means3D, radii, colors, semantic_feature, scales, rotations, scale_modifier, cov3D_precomp,           \
        viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, dL_dout_feature, dL_dout_depth, sh, degree, campos, \
        geomBuffer, R, binningBuffer, imageBuffer, debug

BackwardGrads RasterizeGaussiansBackwardCUDA(BACKWARD_PARAMS) { return backward_grads(BACKWARD_ARGS, nullptr); }

// rasterize_gaussians_backward's 9 gradients + (dL_dviewmatrix [4,4], dL_dprojmatrix [4,4], dL_dcampos [3]), each in the
// layout of its input
using CameraGrads = decltype(std::tuple_cat(BackwardGrads(), std::tuple<torch::Tensor, torch::Tensor, torch::Tensor>()));

// run(camera) -> the 9 gradients, with `camera` the 35 zeroed floats the camera gradient is added to; without `camera`
// run(nullptr), and the three camera gradients are None
template <typename Run>
static CameraGrads with_camera_grads(const torch::Tensor& means3D, const bool camera, const Run& run) {
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor (this build has no CPU path)");
    const c10::cuda::CUDAGuard guard(means3D.device());
    if (!camera) return std::tuple_cat(run(nullptr), std::make_tuple(torch::Tensor(), torch::Tensor(), torch::Tensor()));
    torch::Tensor cam = torch::zeros({F3DGS_CAMERA_GRAD_FLOATS}, means3D.options().dtype(torch::kFloat32));
    return std::tuple_cat(run(cam.data_ptr<float>()),
                          std::make_tuple(cam.narrow(0, 0, 16).view({4, 4}), cam.narrow(0, 16, 16).view({4, 4}),
                                          cam.narrow(0, 32, 3)));
}

// f3dgs_backward_cam / _cam_f16
CameraGrads RasterizeGaussiansBackwardCameraCUDA(BACKWARD_PARAMS) {
    return with_camera_grads(means3D, true, [&](float* cam) { return backward_grads(BACKWARD_ARGS, cam); });
}

// rasterize_gaussians_backward_camera's 12 results, with the feature term of dL/dalpha in the geometric gradients
// (f3dgs_backward_feature_geometry); without `camera` the three camera gradients are None and none is computed
CameraGrads RasterizeGaussiansBackwardFeatureGeometryCUDA(BACKWARD_PARAMS, const bool camera) {
    return with_camera_grads(means3D, camera, [&](float* cam) { return backward_grads(BACKWARD_ARGS, cam, true); });
}

// rasterize_gaussians_backward_feature_geometry's 12 results for the buffers of rasterize_gaussians_antialiased
// (f3dgs_backward_antialiased): the feature term of dL/dalpha only when `features` (the forward's semantic_feature) is
// given, the camera gradients only with `camera`
CameraGrads RasterizeGaussiansBackwardAntialiasedCUDA(BACKWARD_PARAMS, const bool camera,
                                                      const std::optional<torch::Tensor>& features) {
    const torch::Tensor f = features.has_value() ? *features : torch::Tensor();
    return with_camera_grads(means3D, camera,
                             [&](float* cam) { return backward_grads(BACKWARD_ARGS, cam, false, true, f); });
}
// rasterize_gaussians_backward_antialiased's 12 results for the buffers of rasterize_gaussians_alpha_invdepth (or of the
// forward without planes in the same mode), with the gradients of the opacity and inverse-depth planes
// (f3dgs_backward_alpha_invdepth)
CameraGrads RasterizeGaussiansBackwardAlphaInvDepthCUDA(BACKWARD_PARAMS, const torch::Tensor& dL_dout_alpha,
                                                        const torch::Tensor& dL_dout_invdepth, const bool camera,
                                                        const std::optional<torch::Tensor>& features,
                                                        const bool antialiasing) {
    const torch::Tensor f = features.has_value() ? *features : torch::Tensor();
    const torch::Tensor planes[2] = {dL_dout_alpha, dL_dout_invdepth};
    return with_camera_grads(means3D, camera, [&](float* cam) {
        return backward_grads(BACKWARD_ARGS, cam, false, antialiasing, f, planes);
    });
}
#undef BACKWARD_PARAMS
#undef BACKWARD_ARGS

// Accumulating backward for view batches (additive to the reference module): gradients are ADDED into the tensors the
// caller passes (typically views of one flat gradient buffer, see diff_gaussian_rasterization/parallel.py); nothing is
// allocated besides one cached scratch tensor per device.  Undefined / empty tensors stand for "not an input".
// semantic_feature (optional, [P,...,C] float32 or float16): f3dgs_backward_accum_feature_geometry, the feature term of
// dL/dalpha in the geometric gradients.  antialiasing: f3dgs_backward_accum_antialiased, for the buffers of
// rasterize_gaussians_antialiased (with the feature term if semantic_feature is given).  dL_dout_alpha / dL_dout_invdepth
// (optional; one given alone: the other is zero): f3dgs_backward_accum_alpha_invdepth, the gradients of the opacity and
// inverse-depth planes, for the buffers of either forward in the mode `antialiasing`.
void RasterizeGaussiansBackwardAccumCUDA(
    const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii,
    const torch::Tensor& colors, const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier,
    const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
    const float tan_fovx, const float tan_fovy, const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_feature,
    const torch::Tensor& dL_dout_depth, const torch::Tensor& sh, const int degree, const torch::Tensor& campos,
    const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer,
    torch::Tensor scratch, torch::Tensor g_means3D, torch::Tensor g_sh, torch::Tensor g_colors,
    torch::Tensor g_semantic_feature, torch::Tensor g_opacities, torch::Tensor g_scales, torch::Tensor g_rotations,
    torch::Tensor g_cov3D, torch::Tensor g_means2D_out, torch::Tensor grad_accum, torch::Tensor denom,
    const int64_t composite_done_event, const bool debug, const double feature_grad_scale,
    const std::optional<torch::Tensor>& camera_grad, const std::optional<torch::Tensor>& semantic_feature,
    const bool antialiasing, const std::optional<torch::Tensor>& dL_dout_alpha,
    const std::optional<torch::Tensor>& dL_dout_invdepth) {
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor (this build has no CPU path)");
    const c10::cuda::CUDAGuard guard(means3D.device());
    const auto dev = means3D.device();
    const int P = means3D.size(0);
    if (P == 0) return;
    const int H = dL_dout_color.size(1), W = dL_dout_color.size(2);
    int M = 0;
    if (sh.defined() && sh.numel() != 0) M = sh.size(1);
    const int C = (dL_dout_feature.defined() && dL_dout_feature.dim() == 3) ? (int)dL_dout_feature.size(0) : 0;
    auto bg = input(background, dev, "bg"), m3 = input(means3D, dev, "means3D");
    auto col = input(colors, dev, "colors_precomp");
    auto sc = input(scales, dev, "scales"), rot = input(rotations, dev, "rotations");
    auto cov = input(cov3D_precomp, dev, "cov3D_precomp");
    auto vm = input(viewmatrix, dev, "viewmatrix"), pm = input(projmatrix, dev, "projmatrix");
    auto shc = input(sh, dev, "shs"), cp = input(campos, dev, "campos");
    auto gc = input(dL_dout_color, dev, "grad_out_color"), gd = input(dL_dout_depth, dev, "grad_out_depth");
    // a float16 map gradient stands for feature_grad_scale * grad (f3dgs_backward_accum_f16); a float32 one is the
    // gradient itself, so its scale must be 1
    torch::Tensor gf = C ? feature_grad(dL_dout_feature, dev) : torch::Tensor();
    TORCH_CHECK(feature_grad_scale == 1.0 || (gf.defined() && gf.scalar_type() == torch::kFloat16),
                "feature_grad_scale != 1 needs a float16 grad_out_feature (got ",
                gf.defined() ? c10::toString(gf.scalar_type()) : "none", ")");
    TORCH_CHECK(radii.scalar_type() == torch::kInt32 && radii.is_cuda(), "radii must be int32 CUDA");
    auto rad = radii.contiguous();
    const size_t need = f3dgs_backward_scratch_bytes(P);
    TORCH_CHECK(scratch.defined() && scratch.is_cuda() && scratch.scalar_type() == torch::kByte &&
                    scratch.is_contiguous() && (size_t)scratch.numel() >= need,
                "scratch must be a contiguous uint8 CUDA tensor of at least ", need, " bytes");
    // camera_grad (optional): 35 contiguous float32 on the device, ADDED to by the _accum_cam entries
    float* cam = nullptr;
    if (camera_grad.has_value() && camera_grad->defined()) {
        TORCH_CHECK(camera_grad->numel() == F3DGS_CAMERA_GRAD_FLOATS, "camera_grad must have ",
                    F3DGS_CAMERA_GRAD_FLOATS, " elements (got ", camera_grad->numel(), ")");
        cam = in_place(*camera_grad, dev, F3DGS_CAMERA_GRAD_FLOATS, "camera_grad");
    }
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    const bool has_features = semantic_feature.has_value() && semantic_feature->defined();
    const bool has_planes = (dL_dout_alpha.has_value() && dL_dout_alpha->defined()) ||
                            (dL_dout_invdepth.has_value() && dL_dout_invdepth->defined());
    if (has_features || antialiasing || has_planes) {
        torch::Tensor sf;
        if (has_features) {
            check_features(*semantic_feature, dev);
            TORCH_CHECK(semantic_feature->numel() == (int64_t)P * C, "semantic_feature must have P * C = ",
                        (int64_t)P * C, " elements (got ", semantic_feature->numel(), ")");
            sf = semantic_feature->contiguous();
        }
        // the three entries share their arguments up to dL_dcamera; `tail` is the _alpha_invdepth entry's rest
        auto call = [&](auto fn, auto... tail) {
            return fn(P, degree, M, R, C, fptr(bg), W, H, fptr(m3), fptr(shc), fptr(col),
                      C && has_features ? sf.data_ptr() : nullptr,
                      dtype_code(sf), fptr(sc), scale_modifier, fptr(rot), fptr(cov), fptr(vm), fptr(pm), fptr(cp),
                      tan_fovx, tan_fovy, rad.data_ptr<int>(), reinterpret_cast<char*>(geomBuffer.data_ptr()),
                      reinterpret_cast<char*>(binningBuffer.data_ptr()),
                      reinterpret_cast<char*>(imageBuffer.data_ptr()), fptr(gc), gf.defined() ? gf.data_ptr() : nullptr,
                      dtype_code(gf), (float)feature_grad_scale, fptr(gd), reinterpret_cast<char*>(scratch.data_ptr()),
                      in_place(g_opacities, dev, P, "g_opacities"),
                      in_place(g_colors, dev, (int64_t)P * 3, "g_colors_precomp"),
                      in_place(g_semantic_feature, dev, (int64_t)P * C, "g_semantic_feature"),
                      in_place(g_means3D, dev, (int64_t)P * 3, "g_means3D"),
                      in_place(g_cov3D, dev, (int64_t)P * 6, "g_cov3D_precomp"),
                      in_place(g_sh, dev, (int64_t)P * M * 3, "g_sh"),
                      in_place(g_scales, dev, (int64_t)P * 3, "g_scales"),
                      in_place(g_rotations, dev, (int64_t)P * 4, "g_rotations"),
                      in_place(g_means2D_out, dev, (int64_t)P * 3, "g_means2D_out"),
                      in_place(grad_accum, dev, P, "grad_accum"), in_place(denom, dev, P, "denom"),
                      reinterpret_cast<void*>(static_cast<intptr_t>(composite_done_event)), debug ? 1 : 0,
                      (void*)stream, cam, tail...);
        };
        if (has_planes) {
            const torch::Tensor none;
            auto ga = plane_grad(dL_dout_alpha.value_or(none), dev, H, W, "dL_dout_alpha");
            auto gi = plane_grad(dL_dout_invdepth.value_or(none), dev, H, W, "dL_dout_invdepth");
            check_rc(call(f3dgs_backward_accum_alpha_invdepth, antialiasing ? 1 : 0, fptr(ga), fptr(gi)),
                     "f3dgs_backward_accum_alpha_invdepth");
        } else
            check_rc(call(antialiasing ? f3dgs_backward_accum_antialiased : f3dgs_backward_accum_feature_geometry),
                     antialiasing ? "f3dgs_backward_accum_antialiased" : "f3dgs_backward_accum_feature_geometry");
        return;
    }
    // scale: the float16 symbol's scale after the map, () for the float32 one; tail: (dL_dcamera) or ()
    auto run = [&](auto fn, auto gp, auto scale, auto tail) {
        return std::apply(
            fn, std::tuple_cat(
                    std::make_tuple(P, degree, M, R, C, fptr(bg), W, H, fptr(m3), fptr(shc), fptr(col), fptr(sc),
                                    scale_modifier, fptr(rot), fptr(cov), fptr(vm), fptr(pm), fptr(cp), tan_fovx,
                                    tan_fovy, rad.data_ptr<int>(), reinterpret_cast<char*>(geomBuffer.data_ptr()),
                                    reinterpret_cast<char*>(binningBuffer.data_ptr()),
                                    reinterpret_cast<char*>(imageBuffer.data_ptr()), fptr(gc), gp),
                    scale,
                    std::make_tuple(fptr(gd), reinterpret_cast<char*>(scratch.data_ptr()),
                                    in_place(g_opacities, dev, P, "g_opacities"),
                                    in_place(g_colors, dev, (int64_t)P * 3, "g_colors_precomp"),
                                    in_place(g_semantic_feature, dev, (int64_t)P * C, "g_semantic_feature"),
                                    in_place(g_means3D, dev, (int64_t)P * 3, "g_means3D"),
                                    in_place(g_cov3D, dev, (int64_t)P * 6, "g_cov3D_precomp"),
                                    in_place(g_sh, dev, (int64_t)P * M * 3, "g_sh"),
                                    in_place(g_scales, dev, (int64_t)P * 3, "g_scales"),
                                    in_place(g_rotations, dev, (int64_t)P * 4, "g_rotations"),
                                    in_place(g_means2D_out, dev, (int64_t)P * 3, "g_means2D_out"),
                                    in_place(grad_accum, dev, P, "grad_accum"), in_place(denom, dev, P, "denom"),
                                    reinterpret_cast<void*>(static_cast<intptr_t>(composite_done_event)),
                                    debug ? 1 : 0, (void*)stream),
                    tail));
    };
    auto dispatch = [&](auto tail) {
        return [&, tail](auto fn, auto gp) {
            if constexpr (std::is_same_v<decltype(gp), uint16_t*>)
                return run(fn, gp, std::make_tuple((float)feature_grad_scale), tail);
            else
                return run(fn, gp, std::tuple<>(), tail);
        };
    };
    if (cam)
        call_f32_or_f16(gf, f3dgs_backward_accum_cam, "f3dgs_backward_accum_cam", f3dgs_backward_accum_cam_f16,
                        "f3dgs_backward_accum_cam_f16", dispatch(std::make_tuple(cam)));
    else
        call_f32_or_f16(gf, f3dgs_backward_accum, "f3dgs_backward_accum", f3dgs_backward_accum_f16,
                        "f3dgs_backward_accum_f16", dispatch(std::tuple<>()));
}

// Feature lifting (f3dgs_lift_features_accum / _f16): the buffers and R of a forward of this view; feature_map [C,H,W]
// float32 or float16 at the forward's resolution; feature_sum [P,...,C] and weight_sum [P] contiguous float32, ADDED into
void liftFeaturesAccum(const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer,
                       const torch::Tensor& imageBuffer, const torch::Tensor& feature_map, torch::Tensor feature_sum,
                       torch::Tensor weight_sum) {
    TORCH_CHECK(feature_map.is_cuda() && feature_map.dim() == 3 &&
                    (feature_map.scalar_type() == torch::kFloat32 || feature_map.scalar_type() == torch::kFloat16),
                "lift_features_accum: feature_map must be a float32 or float16 CUDA tensor [C,H,W]");
    const auto dev = feature_map.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t C = feature_map.size(0), H = feature_map.size(1), W = feature_map.size(2);
    TORCH_CHECK(C <= INT32_MAX && H <= INT32_MAX && W <= INT32_MAX && weight_sum.numel() <= INT32_MAX,
                "lift_features_accum: sizes too large");
    const int64_t P = weight_sum.numel();
    float* ws = in_place(weight_sum, dev, P, "lift_features_accum: weight_sum");
    float* fs = in_place(feature_sum, dev, P * C, "lift_features_accum: feature_sum");
    for (const torch::Tensor* b : {&geomBuffer, &binningBuffer, &imageBuffer})
        TORCH_CHECK(b->device() == dev && b->scalar_type() == torch::kByte && b->is_contiguous(),
                    "lift_features_accum: the forward buffers must be contiguous uint8 tensors on ", dev);
    if (P == 0) return;
    auto fm = feature_map.contiguous();
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    call_f32_or_f16(fm, f3dgs_lift_features_accum, "f3dgs_lift_features_accum", f3dgs_lift_features_accum_f16,
                    "f3dgs_lift_features_accum_f16", [&](auto fn, auto mp) {
                        return fn((int)P, R, (int)C, (int)W, (int)H, reinterpret_cast<char*>(geomBuffer.data_ptr()),
                                  reinterpret_cast<char*>(binningBuffer.data_ptr()),
                                  reinterpret_cast<char*>(imageBuffer.data_ptr()), mp, fs, ws, (void*)stream);
                    });
}

// Per-Gaussian scores (f3dgs_gaussian_scores_accum): the buffers and R of a forward of this view at width x height;
// weight_sum [P] float32, max_weight [P] float32 (>= 0) and pixel_count [P] int64, contiguous, accumulated in place
void gaussianScoresAccum(const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer,
                         const torch::Tensor& imageBuffer, const int64_t width, const int64_t height,
                         torch::Tensor weight_sum, torch::Tensor max_weight, torch::Tensor pixel_count) {
    TORCH_CHECK(weight_sum.is_cuda(), "gaussian_scores_accum: weight_sum must be a CUDA tensor");
    const auto dev = weight_sum.device();
    const c10::cuda::CUDAGuard guard(dev);
    TORCH_CHECK(weight_sum.numel() <= INT32_MAX && width <= INT32_MAX && height <= INT32_MAX,
                "gaussian_scores_accum: sizes too large");
    const int64_t P = weight_sum.numel();
    float* ws = in_place(weight_sum, dev, P, "gaussian_scores_accum: weight_sum");
    float* mw = in_place(max_weight, dev, P, "gaussian_scores_accum: max_weight");
    TORCH_CHECK(pixel_count.is_cuda() && pixel_count.device() == dev && pixel_count.scalar_type() == torch::kInt64 &&
                    pixel_count.is_contiguous() && pixel_count.numel() == P,
                "gaussian_scores_accum: pixel_count must be a contiguous int64 tensor of ", P, " elements on ", dev);
    for (const torch::Tensor* b : {&geomBuffer, &binningBuffer, &imageBuffer})
        TORCH_CHECK(b->device() == dev && b->scalar_type() == torch::kByte && b->is_contiguous(),
                    "gaussian_scores_accum: the forward buffers must be contiguous uint8 tensors on ", dev);
    if (P == 0) return;
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_gaussian_scores_accum((int)P, R, (int)width, (int)height,
                                         reinterpret_cast<char*>(geomBuffer.data_ptr()),
                                         reinterpret_cast<char*>(binningBuffer.data_ptr()),
                                         reinterpret_cast<char*>(imageBuffer.data_ptr()), ws, mw,
                                         pixel_count.data_ptr<int64_t>(), (void*)stream),
             "f3dgs_gaussian_scores_accum");
}

torch::Tensor markVisible(torch::Tensor& means3D, torch::Tensor& viewmatrix, torch::Tensor& projmatrix) {
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor (this build has no CPU path)");
    const c10::cuda::CUDAGuard guard(means3D.device());
    const auto dev = means3D.device();
    const int P = means3D.size(0);
    torch::Tensor present = torch::full({P}, false, means3D.options().dtype(at::kBool));
    if (P != 0) {
        auto m3 = input(means3D, dev, "means3D"), vm = input(viewmatrix, dev, "viewmatrix"),
             pm = input(projmatrix, dev, "projmatrix");
        cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
        int rc = f3dgs_mark_visible(P, fptr(m3), fptr(vm), fptr(pm), reinterpret_cast<uint8_t*>(present.data_ptr<bool>()),
                                    (void*)stream);
        check_rc(rc, "f3dgs_mark_visible");
    }
    return present;
}

// ---- post-raster feature head (include/f3dgs_b200.h: f3dgs_feature_resize_fwd / _bwd) ----------------------------
namespace {
// a teacher map may be float32 or float16 (the data format's dtype; the float16 symbols upcast it exactly in the kernel)
bool is_target_dtype(const torch::Tensor& t) {
    return t.scalar_type() == torch::kFloat32 || t.scalar_type() == torch::kFloat16;
}
}  // namespace

// -> (out [C,Hg,Wg], loss_sum [1]), float32; with gt: out = sign(resized - gt) * grad_scale and loss_sum =
// sum |resized - gt|.  feature_map and gt may each be float32 or float16 (upcast exactly in the kernel)
std::tuple<torch::Tensor, torch::Tensor> featureResizeFwd(const torch::Tensor& feature_map, const torch::Tensor& gt,
                                                          int64_t Hg, int64_t Wg, double grad_scale) {
    TORCH_CHECK(feature_map.is_cuda() && feature_map.dim() == 3 && is_target_dtype(feature_map),
                "feature_map must be a float32 or float16 CUDA tensor [C,H,W]");
    const c10::cuda::CUDAGuard guard(feature_map.device());
    auto fm = feature_map.contiguous();
    const int C = fm.size(0), H = fm.size(1), W = fm.size(2);
    const bool has_gt = gt.defined() && gt.numel() > 0;
    torch::Tensor g;
    if (has_gt) {
        TORCH_CHECK(gt.is_cuda() && is_target_dtype(gt) && gt.dim() == 3 && gt.size(0) == C && gt.size(1) == Hg &&
                        gt.size(2) == Wg, "gt must be a float32 or float16 CUDA tensor [C,Hg,Wg]");
        g = gt.contiguous();
    }
    auto f32 = fm.options().dtype(torch::kFloat32);
    torch::Tensor out = torch::empty({C, Hg, Wg}, f32);
    torch::Tensor loss = torch::zeros({1}, f32);
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    auto run = [&](auto fn, auto fp, auto gp) {
        return fn(C, H, W, (int)Hg, (int)Wg, fp, gp, (float)grad_scale, out.data_ptr<float>(), loss.data_ptr<float>(),
                  (void*)stream);
    };
    if (fm.scalar_type() == torch::kFloat16) {
        const uint16_t* fp = reinterpret_cast<const uint16_t*>(fm.data_ptr<at::Half>());
        call_f32_or_f16(g, f3dgs_feature_resize_fwd_f16, "f3dgs_feature_resize_fwd_f16",
                        f3dgs_feature_resize_fwd_f16_f16gt, "f3dgs_feature_resize_fwd_f16_f16gt",
                        [&](auto fn, auto gp) { return run(fn, fp, gp); });
    } else {
        call_f32_or_f16(g, f3dgs_feature_resize_fwd, "f3dgs_feature_resize_fwd", f3dgs_feature_resize_fwd_f16gt,
                        "f3dgs_feature_resize_fwd_f16gt", [&](auto fn, auto gp) { return run(fn, fptr(fm), gp); });
    }
    return std::make_tuple(out, loss);
}

// -> dL/dfeature_map [C,H,W] of `dtype`: float32, or float16 holding half_rn(out_scale * the float32 gradient)
torch::Tensor featureResizeBwd(const torch::Tensor& dout, int64_t H, int64_t W, torch::ScalarType dtype,
                               double out_scale) {
    TORCH_CHECK(dout.is_cuda() && dout.dim() == 3 && dout.scalar_type() == torch::kFloat32,
                "dout must be a float32 CUDA tensor [C,Hg,Wg]");
    TORCH_CHECK(dtype == torch::kFloat32 || dtype == torch::kFloat16, "feature_resize_bwd: dtype must be float32 or float16");
    TORCH_CHECK(dtype == torch::kFloat16 || out_scale == 1.0, "feature_resize_bwd: out_scale != 1 needs dtype float16");
    const c10::cuda::CUDAGuard guard(dout.device());
    auto d = dout.contiguous();
    const int C = d.size(0), Hg = d.size(1), Wg = d.size(2);
    torch::Tensor dfm = torch::empty({C, H, W}, d.options().dtype(dtype));
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    call_f32_or_f16(dfm, f3dgs_feature_resize_bwd, "f3dgs_feature_resize_bwd", f3dgs_feature_resize_bwd_f16,
                    "f3dgs_feature_resize_bwd_f16", [&](auto fn, auto op) {
                        if constexpr (std::is_same_v<decltype(op), uint16_t*>)
                            return fn(C, (int)H, (int)W, Hg, Wg, fptr(d), (float)out_scale, op, (void*)stream);
                        else
                            return fn(C, (int)H, (int)W, Hg, Wg, fptr(d), op, (void*)stream);
                    });
    return dfm;
}

// ---- photometric loss (f3dgs_image_loss): image, gt [C,H,W] or [B,C,H,W]
// -> (sums [2] = (sum |image - gt|, sum ssim_map), dL/dimage shaped like image, or an empty tensor without need_grad)
std::tuple<torch::Tensor, torch::Tensor> imageLoss(const torch::Tensor& image, const torch::Tensor& gt, double w_l1,
                                                   double w_ssim, bool need_grad) {
    TORCH_CHECK(image.is_cuda() && image.scalar_type() == torch::kFloat32 && (image.dim() == 3 || image.dim() == 4),
                "image must be a float32 CUDA tensor [C,H,W] or [B,C,H,W]");
    TORCH_CHECK(gt.device() == image.device() && gt.scalar_type() == torch::kFloat32 && gt.sizes() == image.sizes(),
                "gt must be a float32 tensor on ", image.device(), " with the shape of image");
    const c10::cuda::CUDAGuard guard(image.device());
    auto x = image.contiguous(), y = gt.contiguous();
    const int64_t H = x.size(-2), W = x.size(-1);
    TORCH_CHECK(H > 0 && W > 0 && H <= INT32_MAX && W <= INT32_MAX, "image must have H, W >= 1");
    const int64_t planes = x.numel() / (H * W);
    TORCH_CHECK(planes <= INT32_MAX, "too many planes");
    torch::Tensor sums = planes ? torch::empty({2}, x.options()) : torch::zeros({2}, x.options());
    torch::Tensor grad = need_grad ? torch::empty_like(x) : torch::empty({0}, x.options());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_image_loss((int)planes, (int)H, (int)W, fptr(x), fptr(y), (float)w_l1, (float)w_ssim,
                              sums.data_ptr<float>(), need_grad && planes ? grad.data_ptr<float>() : nullptr, (void*)stream),
             "f3dgs_image_loss");
    return std::make_tuple(sums, grad);
}

// ---- feature decoder (f3dgs_decoder_forward / f3dgs_decoder_l1): x [Cin,N] or [Cin,H,W], weight [Cout,Cin] or
// [Cout,Cin,1,1], bias [Cout] or empty (no bias), gt [Cout, <x's spatial shape>]
namespace {
struct DecoderInputs {
    torch::Tensor x, w, b;
    int Cin, Cout, N;
};

DecoderInputs decoder_inputs(const torch::Tensor& x, const torch::Tensor& weight, const torch::Tensor& bias) {
    TORCH_CHECK(x.is_cuda() && x.scalar_type() == torch::kFloat32 && x.dim() >= 2,
                "x must be a float32 CUDA tensor [Cin,N] or [Cin,H,W]");
    const auto dev = x.device();
    TORCH_CHECK(weight.device() == dev && weight.scalar_type() == torch::kFloat32 &&
                    (weight.dim() == 2 || (weight.dim() == 4 && weight.size(2) == 1 && weight.size(3) == 1)),
                "weight must be a float32 tensor [Cout,Cin] or [Cout,Cin,1,1] on ", dev);
    DecoderInputs d;
    d.Cout = (int)weight.size(0);
    d.Cin = (int)weight.size(1);
    TORCH_CHECK(x.size(0) == d.Cin, "x has ", x.size(0), " channels, weight expects Cin = ", d.Cin);
    const int64_t N = x.numel() / std::max<int64_t>(x.size(0), 1);
    TORCH_CHECK(N >= 1 && N <= INT32_MAX, "x must have 1 <= N <= 2^31 - 1 pixels");
    d.N = (int)N;
    const bool has_b = bias.defined() && bias.numel() > 0;
    if (has_b)
        TORCH_CHECK(bias.device() == dev && bias.scalar_type() == torch::kFloat32 && bias.dim() == 1 &&
                        bias.size(0) == d.Cout, "bias must be a float32 tensor [Cout] on ", dev, " (or empty)");
    d.x = x.contiguous();
    d.w = weight.contiguous();
    d.b = has_b ? bias.contiguous() : torch::Tensor();
    return d;
}
}  // namespace

// -> y [Cout, <x's spatial shape>] of dtype float32, or float16 (rounded to nearest even, as y.half())
torch::Tensor decoderForward(const torch::Tensor& x, const torch::Tensor& weight, const torch::Tensor& bias,
                             torch::ScalarType dtype) {
    TORCH_CHECK(dtype == torch::kFloat32 || dtype == torch::kFloat16, "decoder_forward: dtype must be float32 or float16");
    auto d = decoder_inputs(x, weight, bias);
    const c10::cuda::CUDAGuard guard(x.device());
    auto shape = d.x.sizes().vec();
    shape[0] = d.Cout;
    torch::Tensor y = torch::empty(shape, d.x.options().dtype(dtype));
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    call_f32_or_f16(y, f3dgs_decoder_forward, "f3dgs_decoder_forward", f3dgs_decoder_forward_f16,
                    "f3dgs_decoder_forward_f16", [&](auto fn, auto yp) {
                        return fn(d.Cin, d.Cout, d.N, fptr(d.w), fptr(d.b), fptr(d.x), yp, (void*)stream);
                    });
    return y;
}

// -> (loss_sum [1] = sum |y - gt|, dL/dx shaped like x); dweight [Cout,Cin(,1,1)] and dbias [Cout] are ADDED into
std::tuple<torch::Tensor, torch::Tensor> decoderL1(const torch::Tensor& x, const torch::Tensor& gt,
                                                   const torch::Tensor& weight, const torch::Tensor& bias,
                                                   double grad_scale, torch::Tensor dweight, torch::Tensor dbias) {
    auto d = decoder_inputs(x, weight, bias);
    const auto dev = x.device();
    const c10::cuda::CUDAGuard guard(dev);
    TORCH_CHECK(gt.device() == dev && is_target_dtype(gt) && gt.dim() == d.x.dim() && gt.size(0) == d.Cout &&
                    gt.numel() == (int64_t)d.Cout * d.N && gt.sizes().slice(1) == d.x.sizes().slice(1),
                "gt must be a float32 or float16 tensor [Cout, <x's spatial shape>] on ", dev);
    auto g = gt.contiguous();
    float* dw = in_place(dweight, dev, (int64_t)d.Cout * d.Cin, "dweight");
    float* db = in_place(dbias, dev, d.b.defined() ? d.Cout : 0, "dbias");
    torch::Tensor loss = torch::empty({1}, d.x.options());
    torch::Tensor dx = torch::empty_like(d.x);
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    call_f32_or_f16(g, f3dgs_decoder_l1, "f3dgs_decoder_l1", f3dgs_decoder_l1_f16gt, "f3dgs_decoder_l1_f16gt",
                    [&](auto fn, auto gp) {
                        return fn(d.Cin, d.Cout, d.N, fptr(d.w), fptr(d.b), fptr(d.x), gp, (float)grad_scale,
                                  loss.data_ptr<float>(), dx.data_ptr<float>(), dw, db, (void*)stream);
                    });
    return std::make_tuple(loss, dx);
}

// ---- text query (f3dgs_feature_query / _f16x): x [C,N] or [C,H,W] float32 or float16, text [K,D], weight [D,C] or
// [D,C,1,1] or empty (no decoder), bias [D] or empty, positive [K] uint8 / bool or empty
// -> (labels int64, prob float32, logits float32 [K, ...]) shaped like x without its channel axis; an output that is not
// wanted is an empty tensor
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> featureQuery(const torch::Tensor& x, const torch::Tensor& text,
                                                                     const torch::Tensor& weight,
                                                                     const torch::Tensor& bias, double logit_scale,
                                                                     const torch::Tensor& positive, bool want_labels,
                                                                     bool want_prob, bool want_logits) {
    TORCH_CHECK(x.is_cuda() && (x.scalar_type() == torch::kFloat32 || x.scalar_type() == torch::kFloat16) &&
                    x.dim() >= 2, "feature_query: x must be a float32 or float16 CUDA tensor [C,N] or [C,H,W]");
    const auto dev = x.device();
    const c10::cuda::CUDAGuard guard(dev);
    TORCH_CHECK(text.device() == dev && text.scalar_type() == torch::kFloat32 && text.dim() == 2,
                "feature_query: text must be a float32 tensor [K,D] on ", dev);
    const bool has_w = weight.defined() && weight.numel() > 0, has_b = bias.defined() && bias.numel() > 0;
    const bool has_pos = positive.defined() && positive.numel() > 0;
    const int64_t C = x.size(0), K = text.size(0), D = text.size(1);
    if (has_w) {
        TORCH_CHECK(weight.device() == dev && weight.scalar_type() == torch::kFloat32 &&
                        (weight.dim() == 2 || (weight.dim() == 4 && weight.size(2) == 1 && weight.size(3) == 1)) &&
                        weight.size(0) == D && weight.size(1) == C,
                    "feature_query: weight must be a float32 tensor [D,C] or [D,C,1,1] on ", dev, " with D = ", D,
                    " (text) and C = ", C, " (x)");
    } else {
        TORCH_CHECK(D == C, "feature_query: without a decoder text must have x's ", C, " channels (got ", D, ")");
    }
    if (has_b)
        TORCH_CHECK(has_w && bias.device() == dev && bias.scalar_type() == torch::kFloat32 && bias.dim() == 1 &&
                        bias.size(0) == D, "feature_query: bias must be a float32 tensor [D] on ", dev,
                    ", and only with a weight");
    if (has_pos)
        TORCH_CHECK(positive.device() == dev &&
                        (positive.scalar_type() == torch::kUInt8 || positive.scalar_type() == torch::kBool) &&
                        positive.dim() == 1 && positive.size(0) == K,
                    "feature_query: positive must be a uint8 or bool tensor [K] on ", dev);
    TORCH_CHECK(!want_prob || has_pos, "feature_query: prob needs a positive set");
    TORCH_CHECK(want_labels || want_prob || want_logits, "feature_query: no output requested");
    const int64_t N = x.numel() / std::max<int64_t>(C, 1);
    TORCH_CHECK(C >= 1 && K >= 1, "feature_query: x needs a channel and text a prompt");
    TORCH_CHECK(N <= INT32_MAX && C <= INT32_MAX && K <= INT32_MAX && D <= INT32_MAX, "feature_query: sizes too large");
    auto xc = x.contiguous(), tc = text.contiguous();
    auto w = has_w ? weight.contiguous() : torch::Tensor(), b = has_b ? bias.contiguous() : torch::Tensor();
    auto p = has_pos ? positive.contiguous() : torch::Tensor();
    const auto spatial = xc.sizes().slice(1).vec();
    auto lshape = spatial;
    lshape.insert(lshape.begin(), K);
    auto f32 = xc.options().dtype(torch::kFloat32);
    torch::Tensor labels = torch::empty(want_labels ? spatial : std::vector<int64_t>{0}, f32.dtype(torch::kInt64));
    torch::Tensor prob = torch::empty(want_prob ? spatial : std::vector<int64_t>{0}, f32);
    torch::Tensor logits = torch::empty(want_logits ? lshape : std::vector<int64_t>{0}, f32);
    if (N == 0) return std::make_tuple(labels, prob, logits);
    const uint8_t* pp = has_pos ? reinterpret_cast<const uint8_t*>(p.data_ptr()) : nullptr;
    int64_t* lp = want_labels ? labels.data_ptr<int64_t>() : nullptr;
    float* pr = want_prob ? prob.data_ptr<float>() : nullptr;
    float* lg = want_logits ? logits.data_ptr<float>() : nullptr;
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    call_f32_or_f16(xc, f3dgs_feature_query, "f3dgs_feature_query", f3dgs_feature_query_f16x, "f3dgs_feature_query_f16x",
                    [&](auto fn, auto xp) {
                        return fn((int)C, (int)D, (int)K, (int)N, fptr(w), fptr(b), xp, fptr(tc), (float)logit_scale, pp,
                                  lp, pr, lg, (void*)stream);
                    });
    return std::make_tuple(labels, prob, logits);
}

// ---- feature PCA (f3dgs_feature_pca_*): x [C,H,W] or [C,N], a contiguous float32 or float16 CUDA tensor, read in
// place (never copied); mean [C] and components [3,C] contiguous float32, range [2] float32, all on x's device
struct PcaX {
    torch::Tensor x;
    int C, N;
};

PcaX pca_x(const torch::Tensor& x, const char* fn) {
    TORCH_CHECK(x.is_cuda() && (x.scalar_type() == torch::kFloat32 || x.scalar_type() == torch::kFloat16) &&
                    (x.dim() == 2 || x.dim() == 3) && x.is_contiguous(),
                fn, ": x must be a contiguous float32 or float16 CUDA tensor [C,H,W] or [C,N]");
    const int64_t C = x.size(0), N = x.numel() / std::max<int64_t>(C, 1);
    TORCH_CHECK(C >= 3 && C <= 1024 && N >= 7 && N <= INT32_MAX, fn,
                ": needs 3 <= C <= 1024 channels and N >= 7 pixels (at least 3 samples), got C = ", C, ", N = ", N);
    return {x, (int)C, (int)N};
}

torch::Tensor pca_scratch(const PcaX& px) {
    return scratch_tensor(f3dgs_feature_pca_scratch_bytes(px.C, px.N), "f3dgs_feature_pca_scratch_bytes", px.x);
}

// -> (mean [C] float32, cov [C,C] float64)
std::tuple<torch::Tensor, torch::Tensor> featurePcaMoments(const torch::Tensor& x) {
    const PcaX px = pca_x(x, "feature_pca_moments");
    const c10::cuda::CUDAGuard guard(x.device());
    torch::Tensor scratch = pca_scratch(px);
    torch::Tensor mean = torch::empty({px.C}, x.options().dtype(torch::kFloat32));
    torch::Tensor cov = torch::empty({px.C, px.C}, x.options().dtype(torch::kFloat64));
    char* sp = reinterpret_cast<char*>(scratch.data_ptr());
    void* stream = (void*)c10::cuda::getCurrentCUDAStream().stream();
    call_f32_or_f16(x, f3dgs_feature_pca_moments, "f3dgs_feature_pca_moments", f3dgs_feature_pca_moments_f16x,
                    "f3dgs_feature_pca_moments_f16x", [&](auto fn, auto xp) {
                        return fn(px.C, px.N, xp, sp, mean.data_ptr<float>(), cov.data_ptr<double>(), stream);
                    });
    return std::make_tuple(mean, cov);
}

// -> range [2] float32 = (lo, hi)
torch::Tensor featurePcaRange(const torch::Tensor& x, const torch::Tensor& mean, const torch::Tensor& components) {
    const PcaX px = pca_x(x, "feature_pca_range");
    const float* mp = in_place(mean, x.device(), px.C, "feature_pca_range: mean");
    const float* cp = in_place(components, x.device(), 3 * (int64_t)px.C, "feature_pca_range: components");
    const c10::cuda::CUDAGuard guard(x.device());
    torch::Tensor scratch = pca_scratch(px);
    torch::Tensor range = torch::empty({2}, x.options().dtype(torch::kFloat32));
    char* sp = reinterpret_cast<char*>(scratch.data_ptr());
    void* stream = (void*)c10::cuda::getCurrentCUDAStream().stream();
    call_f32_or_f16(x, f3dgs_feature_pca_range, "f3dgs_feature_pca_range", f3dgs_feature_pca_range_f16x,
                    "f3dgs_feature_pca_range_f16x", [&](auto fn, auto xp) {
                        return fn(px.C, px.N, xp, mp, cp, sp, range.data_ptr<float>(), stream);
                    });
    return range;
}

// -> image [H,W,3] or [N,3] float32
torch::Tensor featurePcaImage(const torch::Tensor& x, const torch::Tensor& mean, const torch::Tensor& components,
                              const torch::Tensor& range) {
    const PcaX px = pca_x(x, "feature_pca_image");
    const float* mp = in_place(mean, x.device(), px.C, "feature_pca_image: mean");
    const float* cp = in_place(components, x.device(), 3 * (int64_t)px.C, "feature_pca_image: components");
    const float* rp = in_place(range, x.device(), 2, "feature_pca_image: range");
    const c10::cuda::CUDAGuard guard(x.device());
    auto shape = x.sizes().slice(1).vec();
    shape.push_back(3);
    torch::Tensor image = torch::empty(shape, x.options().dtype(torch::kFloat32));
    void* stream = (void*)c10::cuda::getCurrentCUDAStream().stream();
    call_f32_or_f16(x, f3dgs_feature_pca_image, "f3dgs_feature_pca_image", f3dgs_feature_pca_image_f16x,
                    "f3dgs_feature_pca_image_f16x", [&](auto fn, auto xp) {
                        return fn(px.C, px.N, xp, mp, cp, rp, image.data_ptr<float>(), stream);
                    });
    return image;
}

// ---- initial scales (f3dgs_knn_mean_dist, the reference's simple_knn distCUDA2): points [P,3] -> [P]
torch::Tensor knnMeanDist(const torch::Tensor& points) {
    TORCH_CHECK(points.is_cuda(), "points must be a CUDA tensor (this build has no CPU path)");
    TORCH_CHECK(points.scalar_type() == torch::kFloat32 && points.dim() == 2 && points.size(1) == 3,
                "points must be a float32 tensor [P,3]");
    TORCH_CHECK(points.size(0) <= INT32_MAX, "points: P must be below 2^31");
    const c10::cuda::CUDAGuard guard(points.device());
    auto p = points.contiguous();
    const int P = (int)p.size(0);
    torch::Tensor out = torch::empty({P}, p.options());
    if (P == 0) return out;
    torch::Tensor scratch = scratch_tensor(f3dgs_knn_scratch_bytes(P), "f3dgs_knn_scratch_bytes", p);
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_knn_mean_dist(P, fptr(p), out.data_ptr<float>(), reinterpret_cast<char*>(scratch.data_ptr()),
                                 (void*)stream),
             "f3dgs_knn_mean_dist");
    return out;
}

// ---- densification (f3dgs_densify_plan / f3dgs_densify_apply / f3dgs_reset_opacity)

// -> (scratch, counts): counts = device int32[4] {originals kept, clones kept, children kept per copy, split}
std::tuple<torch::Tensor, torch::Tensor> densifyPlan(const torch::Tensor& grad_accum, const torch::Tensor& denom,
                                                     const torch::Tensor& raw_opacity, const torch::Tensor& raw_scaling,
                                                     double max_grad, double dense_scale, double min_opacity,
                                                     double max_world_scale) {
    TORCH_CHECK(raw_scaling.is_cuda(), "parameters must be CUDA tensors (this build has no CPU path)");
    TORCH_CHECK(raw_scaling.dim() == 2 && raw_scaling.size(1) == 3, "raw_scaling must be [P,3]");
    TORCH_CHECK(raw_scaling.size(0) <= INT32_MAX / 3, "densify: 3 P must be below 2^31");
    const c10::cuda::CUDAGuard guard(raw_scaling.device());
    const auto dev = raw_scaling.device();
    const int P = (int)raw_scaling.size(0);
    auto ga = grad_accum.contiguous(), dn = denom.contiguous();
    const float* gp = in_place(ga, dev, P, "grad_accum");
    const float* dp = in_place(dn, dev, P, "denom");
    const float* op = in_place(raw_opacity, dev, P, "raw_opacity");
    const float* sp = in_place(raw_scaling, dev, 3 * (int64_t)P, "raw_scaling");
    torch::Tensor scratch = scratch_tensor(f3dgs_densify_scratch_bytes(P), "f3dgs_densify_scratch_bytes", raw_scaling);
    torch::Tensor counts = torch::empty({4}, raw_scaling.options().dtype(torch::kInt32));
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_densify_plan(P, gp, dp, op, sp, (float)max_grad, (float)dense_scale, (float)min_opacity,
                                (float)max_world_scale,
                                scratch.numel() ? reinterpret_cast<char*>(scratch.data_ptr()) : nullptr,
                                counts.data_ptr<int32_t>(), (void*)stream),
             "f3dgs_densify_plan");
    return std::make_tuple(scratch, counts);
}

// keep: bool or uint8 [P] CUDA mask -> (scratch, counts): counts = device int32[4] {rows kept, 0, 0, 0}, the plan of a
// densify_apply that keeps the marked rows
std::tuple<torch::Tensor, torch::Tensor> prunePlan(const torch::Tensor& keep) {
    TORCH_CHECK(keep.is_cuda(), "prune_plan: keep must be a CUDA tensor (this build has no CPU path)");
    TORCH_CHECK(keep.dim() == 1 && (keep.scalar_type() == torch::kBool || keep.scalar_type() == torch::kByte),
                "prune_plan: keep must be a bool or uint8 tensor [P]");
    TORCH_CHECK(keep.size(0) <= INT32_MAX / 3, "prune_plan: 3 P must be below 2^31");
    const c10::cuda::CUDAGuard guard(keep.device());
    auto k = keep.contiguous();
    const int P = (int)k.size(0);
    torch::Tensor scratch = scratch_tensor(f3dgs_densify_scratch_bytes(P), "f3dgs_densify_scratch_bytes", k);
    torch::Tensor counts = torch::empty({4}, k.options().dtype(torch::kInt32));
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_prune_plan(P, P ? reinterpret_cast<const uint8_t*>(k.data_ptr()) : nullptr,
                              scratch.numel() ? reinterpret_cast<char*>(scratch.data_ptr()) : nullptr,
                              counts.data_ptr<int32_t>(), (void*)stream),
             "f3dgs_prune_plan");
    return std::make_tuple(scratch, counts);
}

// src / dst: the 21 tensors raw (xyz, f_dc, f_rest, opacity, scaling, rotation, semantic_feature), exp_avg, exp_avg_sq;
// counts: the host copy of densify_plan's counts; dst is written (P' = A + B + 2 Cc rows)
void densifyApply(const torch::Tensor& scratch, const std::vector<int64_t>& counts, const torch::Tensor& normals,
                  const std::vector<torch::Tensor>& src, const std::vector<torch::Tensor>& dst) {
    TORCH_CHECK(src.size() == 21 && dst.size() == 21 && counts.size() == 4, "densify_apply: 21 src, 21 dst, 4 counts");
    TORCH_CHECK(src[0].is_cuda(), "parameters must be CUDA tensors (this build has no CPU path)");
    TORCH_CHECK(src[0].dim() == 2 && src[0].size(1) == 3 && src[0].size(0) <= INT32_MAX / 3, "xyz must be [P,3], 3 P < 2^31");
    TORCH_CHECK(src[2].dim() == 3 && src[6].dim() >= 2, "f_rest must be [P,M-1,3], semantic_feature [P,1,C]");
    const c10::cuda::CUDAGuard guard(src[0].device());
    const auto dev = src[0].device();
    const int64_t P = src[0].size(0), M = 1 + src[2].size(1), C = src[6].size(-1);
    for (int64_t c : counts) TORCH_CHECK(c >= 0 && c <= INT32_MAX, "densify_apply: bad counts");
    const int64_t Pn = counts[0] + counts[1] + 2 * counts[2];
    const int64_t width[7] = {3, 3, 3 * (M - 1), 1, 3, 4, C};
    static const char* names[7] = {"xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic_feature"};
    f3dgs_gaussian_fields f[2][3];
    for (int i = 0; i < 21; i++) {
        for (int k = 0; k < 2; k++) {
            f3dgs_gaussian_fields& g = f[k][i / 7];
            float** slot[7] = {&g.xyz, &g.f_dc, &g.f_rest, &g.opacity, &g.scaling, &g.rotation, &g.semantic_feature};
            *slot[i % 7] = in_place(k ? dst[i] : src[i], dev, (k ? Pn : P) * width[i % 7], names[i % 7]);
        }
    }
    const float* np = in_place(normals, dev, 6 * counts[3], "normals");
    const int32_t c32[4] = {(int32_t)counts[0], (int32_t)counts[1], (int32_t)counts[2], (int32_t)counts[3]};
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_densify_apply((int)P, (int)M, (int)C,
                                 scratch.numel() ? reinterpret_cast<const char*>(scratch.data_ptr()) : nullptr, c32,
                                 np, f[0], f[1], (void*)stream),
             "f3dgs_densify_apply");
}

void resetOpacity(torch::Tensor raw_opacity, torch::Tensor exp_avg, torch::Tensor exp_avg_sq, double ceiling) {
    TORCH_CHECK(raw_opacity.is_cuda(), "parameters must be CUDA tensors (this build has no CPU path)");
    TORCH_CHECK(raw_opacity.numel() <= INT32_MAX, "reset_opacity: P must be below 2^31");
    const auto dev = raw_opacity.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t P = raw_opacity.numel();
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_reset_opacity((int)P, in_place(raw_opacity, dev, P, "raw_opacity"), in_place(exp_avg, dev, P, "exp_avg"),
                                 in_place(exp_avg_sq, dev, P, "exp_avg_sq"), (float)ceiling, (void*)stream),
             "f3dgs_reset_opacity");
}

// ---- fixed-budget densification, 3DGS-MCMC (f3dgs_mcmc_plan / _relocate / _add / _inject_noise)
namespace {
// The 21 tensors raw (xyz, f_dc, f_rest, opacity, scaling, rotation, semantic_feature), exp_avg, exp_avg_sq of `rows`
// rows -> f3dgs_gaussian_fields[3]; M and C are read from the f_rest and semantic_feature shapes of the first group
void gaussian_fields(const std::vector<torch::Tensor>& t, int64_t rows, int64_t M, int64_t C, f3dgs_gaussian_fields f[3]) {
    TORCH_CHECK(t.size() == 21, "21 field tensors expected (raw, exp_avg, exp_avg_sq)");
    const auto dev = t[0].device();
    const int64_t width[7] = {3, 3, 3 * (M - 1), 1, 3, 4, C};
    static const char* names[7] = {"xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic_feature"};
    for (int i = 0; i < 21; i++) {
        f3dgs_gaussian_fields& g = f[i / 7];
        float** slot[7] = {&g.xyz, &g.f_dc, &g.f_rest, &g.opacity, &g.scaling, &g.rotation, &g.semantic_feature};
        *slot[i % 7] = in_place(t[i], dev, rows * width[i % 7], names[i % 7]);
    }
}

// P, M, C of a group of 21 field tensors
std::tuple<int64_t, int64_t, int64_t> field_sizes(const std::vector<torch::Tensor>& t) {
    TORCH_CHECK(t.size() == 21, "21 field tensors expected (raw, exp_avg, exp_avg_sq)");
    TORCH_CHECK(t[0].is_cuda(), "parameters must be CUDA tensors (this build has no CPU path)");
    TORCH_CHECK(t[0].dim() == 2 && t[0].size(1) == 3 && t[0].size(0) <= INT32_MAX / 3, "xyz must be [P,3], 3 P < 2^31");
    TORCH_CHECK(t[2].dim() == 3 && t[6].dim() >= 2, "f_rest must be [P,M-1,3], semantic_feature [P,1,C]");
    return {t[0].size(0), 1 + t[2].size(1), t[6].size(-1)};
}

// A contiguous int32 index tensor on `dev` -> its data (nullptr if empty)
const int32_t* indices(const torch::Tensor& t, const torch::Device& dev, const char* name) {
    TORCH_CHECK(t.is_cuda() && t.device() == dev && t.scalar_type() == torch::kInt32 && t.is_contiguous() && t.dim() == 1,
                name, " must be a contiguous 1-D int32 tensor on ", dev);
    return t.numel() ? t.data_ptr<int32_t>() : nullptr;
}

char* scratch_ptr(const torch::Tensor& scratch) {
    return scratch.numel() ? reinterpret_cast<char*>(scratch.data_ptr()) : nullptr;
}
}  // namespace

// -> (scratch, n_dead device int32[1], index int32[P]: dead ascending then alive ascending, alive_opacity float[P]: the
// first P - n_dead are the alive opacities in index order)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> mcmcPlan(const torch::Tensor& raw_opacity,
                                                                                double min_opacity) {
    TORCH_CHECK(raw_opacity.is_cuda(), "parameters must be CUDA tensors (this build has no CPU path)");
    TORCH_CHECK(raw_opacity.numel() <= INT32_MAX / 3, "mcmc_plan: 3 P must be below 2^31");
    const auto dev = raw_opacity.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int P = (int)raw_opacity.numel();
    const float* op = in_place(raw_opacity, dev, P, "raw_opacity");
    torch::Tensor scratch = scratch_tensor(f3dgs_mcmc_scratch_bytes(P), "f3dgs_mcmc_scratch_bytes", raw_opacity);
    const auto i32 = raw_opacity.options().dtype(torch::kInt32);
    torch::Tensor n_dead = torch::empty({1}, i32), index = torch::empty({P}, i32);
    torch::Tensor alive = torch::empty({P}, raw_opacity.options());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_mcmc_plan(P, op, (float)min_opacity, scratch_ptr(scratch), n_dead.data_ptr<int32_t>(),
                             P ? index.data_ptr<int32_t>() : nullptr, P ? alive.data_ptr<float>() : nullptr,
                             (void*)stream),
             "f3dgs_mcmc_plan");
    return std::make_tuple(scratch, n_dead, index, alive);
}

// fields: the 21 tensors, updated in place; feature_f16: the float16 [P,1,C] copy of the features, or None
void mcmcRelocate(const torch::Tensor& scratch, const torch::Tensor& dead, const torch::Tensor& src, double min_opacity,
                  const std::vector<torch::Tensor>& fields, const c10::optional<torch::Tensor>& feature_f16) {
    const auto [P, M, C] = field_sizes(fields);
    const auto dev = fields[0].device();
    const c10::cuda::CUDAGuard guard(dev);
    TORCH_CHECK(dead.numel() == src.numel(), "mcmc_relocate: dead and src must have the same length");
    f3dgs_gaussian_fields f[3];
    gaussian_fields(fields, P, M, C, f);
    uint16_t* h16 = nullptr;
    if (feature_f16.has_value() && feature_f16->defined() && feature_f16->numel()) {
        const torch::Tensor& h = *feature_f16;
        TORCH_CHECK(h.is_cuda() && h.device() == dev && h.scalar_type() == torch::kFloat16 && h.is_contiguous() &&
                        h.numel() == P * C,
                    "feature_f16 must be a contiguous float16 tensor of ", P * C, " elements on ", dev);
        h16 = reinterpret_cast<uint16_t*>(h.data_ptr<at::Half>());
    }
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_mcmc_relocate((int)P, (int)M, (int)C, (int)dead.numel(), indices(dead, dev, "dead"),
                                 indices(src, dev, "src"), (float)min_opacity, f, h16, scratch_ptr(scratch),
                                 (void*)stream),
             "f3dgs_mcmc_relocate");
}

// src_fields: the 21 tensors of P rows; dst_fields: 21 tensors of P + n rows, written
void mcmcAdd(const torch::Tensor& scratch, const torch::Tensor& src, double min_opacity,
             const std::vector<torch::Tensor>& src_fields, const std::vector<torch::Tensor>& dst_fields) {
    const auto [P, M, C] = field_sizes(src_fields);
    const auto dev = src_fields[0].device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t n = src.numel();
    f3dgs_gaussian_fields s[3], d[3];
    gaussian_fields(src_fields, P, M, C, s);
    gaussian_fields(dst_fields, P + n, M, C, d);
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_mcmc_add((int)P, (int)M, (int)C, (int)n, indices(src, dev, "src"), (float)min_opacity, s, d,
                            scratch_ptr(scratch), (void*)stream),
             "f3dgs_mcmc_add");
}

// xyz [P,3] in place; eps [P,3] the normals
void mcmcInjectNoise(torch::Tensor xyz, const torch::Tensor& raw_opacity, const torch::Tensor& raw_scaling,
                     const torch::Tensor& raw_rotation, const torch::Tensor& eps, double scale) {
    TORCH_CHECK(xyz.is_cuda(), "parameters must be CUDA tensors (this build has no CPU path)");
    TORCH_CHECK(xyz.dim() == 2 && xyz.size(1) == 3 && xyz.size(0) <= INT32_MAX / 4, "xyz must be [P,3], 4 P < 2^31");
    const auto dev = xyz.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t P = xyz.size(0);
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_mcmc_inject_noise((int)P, in_place(xyz, dev, 3 * P, "xyz"), in_place(raw_opacity, dev, P, "raw_opacity"),
                                     in_place(raw_scaling, dev, 3 * P, "raw_scaling"),
                                     in_place(raw_rotation, dev, 4 * P, "raw_rotation"), in_place(eps, dev, 3 * P, "eps"),
                                     (float)scale, (void*)stream),
             "f3dgs_mcmc_inject_noise");
}

// ---- 3D smoothing filter, Mip-Splatting (f3dgs_filter3d_compute / _apply / _apply_backward,
// f3dgs_reset_opacity_filter3d)
namespace {
// An optional output of `numel` float32 elements shaped like `like`: the caller's tensor, or a new one
torch::Tensor output_or_new(const c10::optional<torch::Tensor>& t, const torch::Tensor& like, const char* name) {
    if (!t.has_value() || !t->defined()) return torch::empty_like(like, torch::MemoryFormat::Contiguous);
    in_place(*t, like.device(), like.numel(), name);
    return *t;
}
}  // namespace

// means3D [P,3], viewmatrices [V,4,4] (or [V,16]), intrinsics [V,4] = (fx, fy, W, H) -> (filter [P,1], n_seen device
// int32[1])
std::tuple<torch::Tensor, torch::Tensor> filter3dCompute(const torch::Tensor& means3D, const torch::Tensor& viewmatrices,
                                                         const torch::Tensor& intrinsics) {
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor (this build has no CPU path)");
    TORCH_CHECK(means3D.dim() == 2 && means3D.size(1) == 3 && means3D.size(0) <= INT32_MAX / 3,
                "means3D must be [P,3], 3 P < 2^31");
    const auto dev = means3D.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t P = means3D.size(0), V = intrinsics.dim() == 2 ? intrinsics.size(0) : -1;
    TORCH_CHECK(V >= 1 && intrinsics.size(1) == 4 && viewmatrices.numel() == 16 * V,
                "filter3d_compute: intrinsics must be [V,4] and viewmatrices [V,4,4] with V >= 1");
    auto m = input(means3D, dev, "means3D"), vm = input(viewmatrices, dev, "viewmatrices");
    auto in = input(intrinsics, dev, "intrinsics");
    torch::Tensor filter = torch::empty({P, 1}, m.options());
    torch::Tensor n_seen = torch::zeros({1}, m.options().dtype(torch::kInt32));
    if (P == 0) return std::make_tuple(filter, n_seen);
    torch::Tensor scratch = torch::empty({(int64_t)f3dgs_filter3d_scratch_bytes((int)P)}, m.options().dtype(torch::kUInt8));
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_filter3d_compute((int)P, (int)V, fptr(m), fptr(vm), fptr(in), filter.data_ptr<float>(),
                                    n_seen.data_ptr<int32_t>(), scratch_ptr(scratch), (void*)stream),
             "f3dgs_filter3d_compute");
    return std::make_tuple(filter, n_seen);
}

// opacity [P,1], scales [P,3], filter [P,1] -> (opacity_out, scales_out), written into the given tensors or new ones
std::tuple<torch::Tensor, torch::Tensor> filter3dApply(const torch::Tensor& opacity, const torch::Tensor& scales,
                                                       const torch::Tensor& filter,
                                                       const c10::optional<torch::Tensor>& opacity_out,
                                                       const c10::optional<torch::Tensor>& scales_out) {
    TORCH_CHECK(scales.is_cuda(), "scales must be a CUDA tensor (this build has no CPU path)");
    TORCH_CHECK(scales.dim() == 2 && scales.size(1) == 3 && scales.size(0) <= INT32_MAX / 3,
                "scales must be [P,3], 3 P < 2^31");
    const auto dev = scales.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t P = scales.size(0);
    TORCH_CHECK(opacity.numel() == P && filter.numel() == P, "filter3d_apply: opacity and filter must have P elements");
    auto o = input(opacity, dev, "opacity"), s = input(scales, dev, "scales"), f = input(filter, dev, "filter");
    torch::Tensor oo = output_or_new(opacity_out, o, "opacity_out"), so = output_or_new(scales_out, s, "scales_out");
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_filter3d_apply((int)P, fptr(o), fptr(s), fptr(f), P ? oo.data_ptr<float>() : nullptr,
                                  P ? so.data_ptr<float>() : nullptr, (void*)stream),
             "f3dgs_filter3d_apply");
    return std::make_tuple(oo, so);
}

// -> (dL_dopacity, dL_dscales) from the gradients of the filtered tensors; written into the given tensors (which may be
// the filtered gradients themselves: in place) or new ones
std::tuple<torch::Tensor, torch::Tensor> filter3dApplyBackward(const torch::Tensor& opacity, const torch::Tensor& scales,
                                                               const torch::Tensor& filter,
                                                               const torch::Tensor& dL_dopacity_f,
                                                               const torch::Tensor& dL_dscales_f,
                                                               const c10::optional<torch::Tensor>& dL_dopacity,
                                                               const c10::optional<torch::Tensor>& dL_dscales) {
    TORCH_CHECK(scales.is_cuda(), "scales must be a CUDA tensor (this build has no CPU path)");
    TORCH_CHECK(scales.dim() == 2 && scales.size(1) == 3 && scales.size(0) <= INT32_MAX / 3,
                "scales must be [P,3], 3 P < 2^31");
    const auto dev = scales.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t P = scales.size(0);
    TORCH_CHECK(opacity.numel() == P && filter.numel() == P && dL_dopacity_f.numel() == P &&
                    dL_dscales_f.numel() == 3 * P,
                "filter3d_apply_backward: opacity, filter and dL_dopacity_f must have P elements, dL_dscales_f 3 P");
    auto o = input(opacity, dev, "opacity"), s = input(scales, dev, "scales"), f = input(filter, dev, "filter");
    // an in-place output must be the caller's contiguous tensor itself, so the upstream gradients are not copied then
    const bool go_in_place = dL_dopacity.has_value() && dL_dopacity->defined() && dL_dopacity->is_same(dL_dopacity_f);
    const bool gs_in_place = dL_dscales.has_value() && dL_dscales->defined() && dL_dscales->is_same(dL_dscales_f);
    auto gof = go_in_place ? dL_dopacity_f : input(dL_dopacity_f, dev, "dL_dopacity_f");
    auto gsf = gs_in_place ? dL_dscales_f : input(dL_dscales_f, dev, "dL_dscales_f");
    torch::Tensor go = output_or_new(dL_dopacity, gof, "dL_dopacity"), gs = output_or_new(dL_dscales, gsf, "dL_dscales");
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_filter3d_apply_backward((int)P, fptr(o), fptr(s), fptr(f), fptr(gof), fptr(gsf),
                                           P ? go.data_ptr<float>() : nullptr, P ? gs.data_ptr<float>() : nullptr,
                                           (void*)stream),
             "f3dgs_filter3d_apply_backward");
    return std::make_tuple(go, gs);
}

void resetOpacityFilter3d(torch::Tensor raw_opacity, const torch::Tensor& raw_scaling, const torch::Tensor& filter,
                          torch::Tensor exp_avg, torch::Tensor exp_avg_sq, double ceiling) {
    TORCH_CHECK(raw_opacity.is_cuda(), "parameters must be CUDA tensors (this build has no CPU path)");
    TORCH_CHECK(raw_opacity.numel() <= INT32_MAX / 3, "reset_opacity_filter3d: 3 P must be below 2^31");
    const auto dev = raw_opacity.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t P = raw_opacity.numel();
    auto s = input(raw_scaling, dev, "raw_scaling"), f = input(filter, dev, "filter");
    TORCH_CHECK(raw_scaling.numel() == 3 * P && filter.numel() == P,
                "reset_opacity_filter3d: raw_scaling must have 3 P elements and filter P");
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_reset_opacity_filter3d((int)P, in_place(raw_opacity, dev, P, "raw_opacity"), fptr(s), fptr(f),
                                          in_place(exp_avg, dev, P, "exp_avg"), in_place(exp_avg_sq, dev, P, "exp_avg_sq"),
                                          (float)ceiling, (void*)stream),
             "f3dgs_reset_opacity_filter3d");
}

// ---- activation prologue + fused optimizer step (f3dgs_activate / f3dgs_adam_step): in-place on the caller's tensors
void activateParams(const torch::Tensor& raw_opacity, const torch::Tensor& raw_scaling, const torch::Tensor& raw_rotation,
                    const torch::Tensor& f_dc, const torch::Tensor& f_rest, torch::Tensor opacity, torch::Tensor scales,
                    torch::Tensor rotations, torch::Tensor shs) {
    TORCH_CHECK(raw_opacity.is_cuda(), "parameters must be CUDA tensors (this build has no CPU path)");
    const auto dev = raw_opacity.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t P = raw_opacity.size(0);
    const int M = shs.defined() && shs.numel() ? (int)shs.size(1) : 0;
    auto ro = input(raw_opacity, dev, "raw_opacity"), rs = input(raw_scaling, dev, "raw_scaling");
    auto rr = input(raw_rotation, dev, "raw_rotation"), dc = input(f_dc, dev, "f_dc"), rest = input(f_rest, dev, "f_rest");
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check_rc(f3dgs_activate((int)P, M, fptr(ro), fptr(rs), fptr(rr), fptr(dc), fptr(rest),
                            in_place(opacity, dev, P, "opacity"), in_place(scales, dev, 3 * P, "scales"),
                            in_place(rotations, dev, 4 * P, "rotations"), in_place(shs, dev, 3 * M * P, "shs"),
                            (void*)stream),
             "f3dgs_activate");
}

// param_f16 (optional, IDENTITY groups): a contiguous float16 tensor of param's size, written with param.half() after
// the step (f3dgs_adam_step_f16out).  visible (optional): a contiguous bool or uint8 tensor of P elements on param's
// device; only the rows it marks (P rows of numel / P elements) are stepped (f3dgs_adam_step_masked[_f16out])
void adamStep(int64_t kind, torch::Tensor param, const torch::Tensor& grad_activated, torch::Tensor exp_avg,
              torch::Tensor exp_avg_sq, int64_t M, double lr, double beta1, double beta2, double eps, int64_t step,
              const c10::optional<torch::Tensor>& param_f16, const c10::optional<torch::Tensor>& visible) {
    TORCH_CHECK(param.is_cuda(), "parameters must be CUDA tensors (this build has no CPU path)");
    const auto dev = param.device();
    const c10::cuda::CUDAGuard guard(dev);
    const int64_t n = param.numel();
    auto g = input(grad_activated, dev, "grad_activated");
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    float* p = in_place(param, dev, n, "param");
    float *m = in_place(exp_avg, dev, n, "exp_avg"), *v = in_place(exp_avg_sq, dev, n, "exp_avg_sq");
    uint16_t* h16 = nullptr;
    if (param_f16.has_value() && param_f16->defined()) {
        const torch::Tensor& h = *param_f16;
        TORCH_CHECK(h.is_cuda() && h.device() == dev && h.scalar_type() == torch::kFloat16 && h.is_contiguous() &&
                        h.numel() == n,
                    "param_f16 must be a contiguous float16 tensor of ", n, " elements on ", dev);
        h16 = reinterpret_cast<uint16_t*>(h.data_ptr<at::Half>());
    }
    if (visible.has_value() && visible->defined()) {
        const torch::Tensor& mask = *visible;
        TORCH_CHECK(mask.is_cuda() && mask.device() == dev &&
                        (mask.scalar_type() == torch::kBool || mask.scalar_type() == torch::kByte) &&
                        mask.is_contiguous() && mask.numel() <= INT32_MAX,
                    "visible must be a contiguous bool or uint8 tensor of P < 2^31 elements on ", dev);
        const int P = (int)mask.numel();
        const uint8_t* vis = P ? reinterpret_cast<const uint8_t*>(mask.data_ptr()) : nullptr;
        if (h16)
            check_rc(f3dgs_adam_step_masked_f16out((int)kind, (size_t)n, P, (int)M, p, fptr(g), m, v, vis, h16,
                                                   (float)lr, (float)beta1, (float)beta2, (float)eps, (int)step,
                                                   (void*)stream),
                     "f3dgs_adam_step_masked_f16out");
        else
            check_rc(f3dgs_adam_step_masked((int)kind, (size_t)n, P, (int)M, p, fptr(g), m, v, vis, (float)lr,
                                            (float)beta1, (float)beta2, (float)eps, (int)step, (void*)stream),
                     "f3dgs_adam_step_masked");
        return;
    }
    if (h16) {
        check_rc(f3dgs_adam_step_f16out((int)kind, (size_t)n, (int)M, p, fptr(g), m, v, h16, (float)lr, (float)beta1,
                                        (float)beta2, (float)eps, (int)step, (void*)stream),
                 "f3dgs_adam_step_f16out");
        return;
    }
    check_rc(f3dgs_adam_step((int)kind, (size_t)n, (int)M, p, fptr(g), m, v, (float)lr, (float)beta1, (float)beta2,
                             (float)eps, (int)step, (void*)stream),
             "f3dgs_adam_step");
}

// Read-only views into the opaque buffers for the parity harness (not part of the reference API).
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> debugViews(
    const torch::Tensor& geomBuffer, const torch::Tensor& binningBuffer, const torch::Tensor& imgBuffer, int P,
    int W, int H, int R) {
    f3dgs_layout L;
    check_rc(f3dgs_get_layout(P, W, H, R, &L), "f3dgs_get_layout");
    const int64_t tiles = (int64_t)((W + 15) / 16) * ((H + 15) / 16);
    auto dev = geomBuffer.device();
    auto view = [&](const torch::Tensor& buf, size_t off, int64_t count, torch::ScalarType ty, int64_t esize) {
        auto bytes = buf.narrow(0, (int64_t)off, count * esize);
        return bytes.view(ty).clone();
    };
    torch::Tensor point_list = R ? view(binningBuffer, L.bin_point_list, R, torch::kInt32, 4)
                                 : torch::empty({0}, torch::TensorOptions().dtype(torch::kInt32).device(dev));
    torch::Tensor ranges = view(imgBuffer, L.img_ranges, tiles * 2, torch::kInt32, 4).view({tiles, 2});
    torch::Tensor n_contrib = view(imgBuffer, L.img_n_contrib, (int64_t)W * H, torch::kInt32, 4).view({H, W});
    torch::Tensor final_T = view(imgBuffer, L.img_final_T, (int64_t)W * H, torch::kFloat32, 4).view({H, W});
    torch::Tensor rec = view(geomBuffer, L.geom_rec, (int64_t)P * 12, torch::kFloat32, 4).view({P, 12});
    return std::make_tuple(point_list, ranges, n_contrib, final_T, rec);
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.def("rasterize_gaussians", &RasterizeGaussiansCUDA);
    m.def("rasterize_gaussians_backward", &RasterizeGaussiansBackwardCUDA);
    m.def("mark_visible", &markVisible);
    {
        namespace py = pybind11;
        m.def("rasterize_gaussians_backward_accum", &RasterizeGaussiansBackwardAccumCUDA, py::arg("background"),
              py::arg("means3D"), py::arg("radii"), py::arg("colors"), py::arg("scales"), py::arg("rotations"),
              py::arg("scale_modifier"), py::arg("cov3D_precomp"), py::arg("viewmatrix"), py::arg("projmatrix"),
              py::arg("tan_fovx"), py::arg("tan_fovy"), py::arg("dL_dout_color"), py::arg("dL_dout_feature"),
              py::arg("dL_dout_depth"), py::arg("sh"), py::arg("degree"), py::arg("campos"), py::arg("geomBuffer"),
              py::arg("R"), py::arg("binningBuffer"), py::arg("imageBuffer"), py::arg("scratch"), py::arg("g_means3D"),
              py::arg("g_sh"), py::arg("g_colors"), py::arg("g_semantic_feature"), py::arg("g_opacities"),
              py::arg("g_scales"), py::arg("g_rotations"), py::arg("g_cov3D"), py::arg("g_means2D_out"),
              py::arg("grad_accum"), py::arg("denom"), py::arg("composite_done_event"), py::arg("debug"),
              py::arg("feature_grad_scale") = 1.0, py::arg("camera_grad") = py::none(),
              py::arg("semantic_feature") = py::none(), py::arg("antialiasing") = false,
              py::arg("dL_dout_alpha") = py::none(), py::arg("dL_dout_invdepth") = py::none());
        m.def("rasterize_gaussians_antialiased", &RasterizeGaussiansAntialiasedCUDA);
        m.def("rasterize_gaussians_backward_antialiased", &RasterizeGaussiansBackwardAntialiasedCUDA,
              py::arg("background"), py::arg("means3D"), py::arg("radii"), py::arg("colors"), py::arg("features_like"),
              py::arg("scales"), py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"),
              py::arg("viewmatrix"), py::arg("projmatrix"), py::arg("tan_fovx"), py::arg("tan_fovy"),
              py::arg("dL_dout_color"), py::arg("dL_dout_feature"), py::arg("dL_dout_depth"), py::arg("sh"),
              py::arg("degree"), py::arg("campos"), py::arg("geomBuffer"), py::arg("R"), py::arg("binningBuffer"),
              py::arg("imageBuffer"), py::arg("debug"), py::arg("camera") = false,
              py::arg("semantic_feature") = py::none());
        m.def("rasterize_gaussians_alpha_invdepth", &RasterizeGaussiansAlphaInvDepthCUDA, py::arg("background"),
              py::arg("means3D"), py::arg("colors"), py::arg("semantic_feature"), py::arg("opacity"), py::arg("scales"),
              py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"), py::arg("viewmatrix"),
              py::arg("projmatrix"), py::arg("tan_fovx"), py::arg("tan_fovy"), py::arg("image_height"),
              py::arg("image_width"), py::arg("sh"), py::arg("degree"), py::arg("campos"), py::arg("prefiltered"),
              py::arg("debug"), py::arg("antialiasing") = false);
        m.def("rasterize_gaussians_backward_alpha_invdepth", &RasterizeGaussiansBackwardAlphaInvDepthCUDA,
              py::arg("background"), py::arg("means3D"), py::arg("radii"), py::arg("colors"), py::arg("features_like"),
              py::arg("scales"), py::arg("rotations"), py::arg("scale_modifier"), py::arg("cov3D_precomp"),
              py::arg("viewmatrix"), py::arg("projmatrix"), py::arg("tan_fovx"), py::arg("tan_fovy"),
              py::arg("dL_dout_color"), py::arg("dL_dout_feature"), py::arg("dL_dout_depth"), py::arg("sh"),
              py::arg("degree"), py::arg("campos"), py::arg("geomBuffer"), py::arg("R"), py::arg("binningBuffer"),
              py::arg("imageBuffer"), py::arg("debug"), py::arg("dL_dout_alpha"), py::arg("dL_dout_invdepth"),
              py::arg("camera") = false, py::arg("semantic_feature") = py::none(), py::arg("antialiasing") = false);
    }
    m.def("rasterize_gaussians_backward_camera", &RasterizeGaussiansBackwardCameraCUDA);
    m.def("rasterize_gaussians_backward_feature_geometry", &RasterizeGaussiansBackwardFeatureGeometryCUDA);
    m.def("lift_features_accum", &liftFeaturesAccum, pybind11::arg("geomBuffer"), pybind11::arg("R"),
          pybind11::arg("binningBuffer"), pybind11::arg("imageBuffer"), pybind11::arg("feature_map"),
          pybind11::arg("feature_sum"), pybind11::arg("weight_sum"));
    m.def("gaussian_scores_accum", &gaussianScoresAccum, pybind11::arg("geomBuffer"), pybind11::arg("R"),
          pybind11::arg("binningBuffer"), pybind11::arg("imageBuffer"), pybind11::arg("width"), pybind11::arg("height"),
          pybind11::arg("weight_sum"), pybind11::arg("max_weight"), pybind11::arg("pixel_count"));
    m.def("feature_resize_fwd", &featureResizeFwd);
    m.def("feature_resize_bwd", &featureResizeBwd, pybind11::arg("dout"), pybind11::arg("H"), pybind11::arg("W"),
          pybind11::arg("dtype") = torch::kFloat32, pybind11::arg("out_scale") = 1.0);
    m.def("image_loss", &imageLoss);
    m.def("decoder_forward", &decoderForward, pybind11::arg("x"), pybind11::arg("weight"), pybind11::arg("bias"),
          pybind11::arg("dtype") = torch::kFloat32);
    m.def("decoder_l1", &decoderL1);
    m.def("feature_query", &featureQuery, pybind11::arg("x"), pybind11::arg("text"), pybind11::arg("weight"),
          pybind11::arg("bias"), pybind11::arg("logit_scale"), pybind11::arg("positive"), pybind11::arg("want_labels"),
          pybind11::arg("want_prob"), pybind11::arg("want_logits"));
    m.def("feature_pca_moments", &featurePcaMoments);
    m.def("feature_pca_range", &featurePcaRange);
    m.def("feature_pca_image", &featurePcaImage);
    m.def("knn_mean_dist", &knnMeanDist);
    m.def("densify_plan", &densifyPlan);
    m.def("densify_apply", &densifyApply);
    m.def("prune_plan", &prunePlan, pybind11::arg("keep"));
    m.def("reset_opacity", &resetOpacity, pybind11::arg("raw_opacity"), pybind11::arg("exp_avg"),
          pybind11::arg("exp_avg_sq"), pybind11::arg("ceiling") = 0.01);
    m.def("mcmc_plan", &mcmcPlan, pybind11::arg("raw_opacity"), pybind11::arg("min_opacity"));
    m.def("mcmc_relocate", &mcmcRelocate, pybind11::arg("scratch"), pybind11::arg("dead"), pybind11::arg("src"),
          pybind11::arg("min_opacity"), pybind11::arg("fields"), pybind11::arg("feature_f16") = pybind11::none());
    m.def("mcmc_add", &mcmcAdd, pybind11::arg("scratch"), pybind11::arg("src"), pybind11::arg("min_opacity"),
          pybind11::arg("src_fields"), pybind11::arg("dst_fields"));
    m.def("mcmc_inject_noise", &mcmcInjectNoise, pybind11::arg("xyz"), pybind11::arg("raw_opacity"),
          pybind11::arg("raw_scaling"), pybind11::arg("raw_rotation"), pybind11::arg("eps"), pybind11::arg("scale"));
    m.def("filter3d_compute", &filter3dCompute, pybind11::arg("means3D"), pybind11::arg("viewmatrices"),
          pybind11::arg("intrinsics"));
    m.def("filter3d_apply", &filter3dApply, pybind11::arg("opacity"), pybind11::arg("scales"), pybind11::arg("filter"),
          pybind11::arg("opacity_out") = pybind11::none(), pybind11::arg("scales_out") = pybind11::none());
    m.def("filter3d_apply_backward", &filter3dApplyBackward, pybind11::arg("opacity"), pybind11::arg("scales"),
          pybind11::arg("filter"), pybind11::arg("dL_dopacity_f"), pybind11::arg("dL_dscales_f"),
          pybind11::arg("dL_dopacity") = pybind11::none(), pybind11::arg("dL_dscales") = pybind11::none());
    m.def("reset_opacity_filter3d", &resetOpacityFilter3d, pybind11::arg("raw_opacity"), pybind11::arg("raw_scaling"),
          pybind11::arg("filter"), pybind11::arg("exp_avg"), pybind11::arg("exp_avg_sq"), pybind11::arg("ceiling") = 0.01);
    m.def("activate", &activateParams);
    m.def("adam_step", &adamStep, pybind11::arg("kind"), pybind11::arg("param"), pybind11::arg("grad_activated"),
          pybind11::arg("exp_avg"), pybind11::arg("exp_avg_sq"), pybind11::arg("M"), pybind11::arg("lr"),
          pybind11::arg("beta1"), pybind11::arg("beta2"), pybind11::arg("eps"), pybind11::arg("step"),
          pybind11::arg("param_f16") = pybind11::none(), pybind11::arg("visible") = pybind11::none());
    m.def("backward_scratch_bytes", [](int P) { return (unsigned long long)f3dgs_backward_scratch_bytes(P); });
    m.def("debug_views", &debugViews);
    m.def("launch_count", []() { return (unsigned long long)f3dgs_launch_count(); });
    m.def("abi_version", []() { return f3dgs_abi_version(); });
    m.def("profile_enable", [](bool on) { f3dgs_profile_enable(on ? 1 : 0); });
    m.def("profile_read", []() {
        std::vector<double> ms(F3DGS_N_STAGES, 0.0);
        std::vector<unsigned long long> cnt(F3DGS_N_STAGES, 0);
        check_rc(f3dgs_profile_read(ms.data(), cnt.data()), "f3dgs_profile_read");
        return std::make_pair(ms, cnt);
    });
}
