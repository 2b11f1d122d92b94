// Internal launch interface between the C-ABI orchestration (api.cu) and the kernel TUs.  A launcher templated on the
// element type of its data is instantiated for float and __half in its .cu.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "common.cuh"

namespace f3dgs {

extern std::atomic<unsigned long long> g_launches;  // kernels launched by this library (api.cu)

struct ViewParams {
    int P, D, M, C;
    int W, H;
    uint32_t grid_x, grid_y;
    float tan_fovx, tan_fovy, focal_x, focal_y;
    float scale_modifier;
    const float* viewmatrix;
    const float* projmatrix;
    const float* cam_pos;
};

// ---- preprocess.cu
void launch_preprocess_fwd(const ViewParams& vp, const float* means3D, const float* scales,
                           const float* rotations, const float* opacities, const float* shs,
                           const float* cov3D_precomp, const float* colors_precomp, bool prefiltered,
                           int* radii, SplatRec* rec, float* cov3D, uint8_t* clamped,
                           uint32_t* tiles_touched, cudaStream_t s, bool antialiasing = false);

// dL_dcamera (optional, 35 floats: dL/dviewmatrix [16], dL/dprojmatrix [16], dL/dcampos [3]) is ADDED to.  Its
// float64 block partials come from the default memory pool: cudaErrorMemoryAllocation if that fails.
// antialiasing: the backward of an antialiased forward, whose records `rec` hold op_eff = opacity * rho.  dL_dop_eff
// [P] is the composite's dL/dop_eff; dL_dopacity gets rho * dL_dop_eff (assigned, or added with `accumulate`).  In the
// assigning backward the two may be one buffer, rescaled in place.
cudaError_t launch_preprocess_bwd(const ViewParams& vp, const float* means3D, const int* radii, const float* shs,
                                  const uint8_t* clamped, const float* scales, const float* rotations,
                                  const float* cov3D, const float* dL_dmean2D, const float* dL_dconic,
                                  float* dL_dmean3D, const float* dL_dcolor, float* dL_dcov3D, float* dL_dsh,
                                  float* dL_dscale, float* dL_drot, const float* dL_dz, cudaStream_t s,
                                  bool accumulate = false, float* grad_accum = nullptr, float* denom = nullptr,
                                  float* dL_dcamera = nullptr, bool antialiasing = false, const SplatRec* rec = nullptr,
                                  const float* dL_dop_eff = nullptr, float* dL_dopacity = nullptr);

void launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                         cudaStream_t s);

// ---- binning.cu
void launch_duplicate_keys(int P, const SplatRec* rec, const uint32_t* offsets, const int* radii,
                           uint32_t grid_x, uint32_t grid_y, uint64_t* keys, uint32_t* values,
                           cudaStream_t s);
void launch_tile_ranges(int R, const uint64_t* sorted_keys, uint2* ranges, cudaStream_t s);

// ---- composite_fwd.cu
// returns cudaSuccess or the launch error.  TF (float or __half) is the element type of features and out_feature: the
// float16 map is bitwise the float32 map of the exactly upcast features rounded to nearest even.  With out_alpha (then
// out_invdepth too, both [H,W]): also the opacity plane 1 - final_T and the inverse-depth plane sum_i w_i / z_i; every
// other output is bitwise that of the call without them
template <typename TF>
cudaError_t launch_composite_fwd(const ViewParams& vp, const uint2* ranges, const uint32_t* point_list,
                                 const SplatRec* rec, const TF* features, const float* bg,
                                 float* final_T, uint32_t* n_contrib, float* out_color,
                                 TF* out_feature, float* out_depth, int* counters, cudaStream_t s,
                                 float* out_alpha = nullptr, float* out_invdepth = nullptr);

// ---- composite_bwd.cu + feature_bwd.cu: the composite backward of a view, from that view's forward buffers
struct ForwardBuffers {
    const uint2* ranges;
    const uint32_t* point_list;
    const SplatRec* rec;
    const float* final_T;
    const uint32_t* n_contrib;
    int* counters;  // the image buffer's work-counter region
    int R;
};
// The Gaussians' feature rows [P, C], float32 or float16 (upcast exactly, as the forward reads them); rows == nullptr:
// none given
struct FeatureRows {
    const void* rows = nullptr;
    bool f16 = false;
};
// Geometric gradients from a kernel at two CTAs per SM.  With C > 0 and R > 0 that kernel also emits per-(tile, block)
// instance lists (scratch of the device's default pool, freed on the stream before return), and a second kernel forms
// dL_dfeature from them.  TG (float or __half) is the element type of dL_dfeat_pix; a __half map stands for
// dL/dO = scale * float(h) (the scale is not read for a float map).  With feat.rows (and C > 0, R > 0) the feature term
// of dL/dalpha is added to dL_dmean2D, dL_dconic and dL_dopacity by two more kernels over the same lists.  With
// dL_dalpha (then dL_dinvdepth too, both [H,W]): the gradients of the forward's opacity and inverse-depth planes join
// dL/dalpha and dL_dz in the same geometry walk; with both zero every output is bitwise that of the call without them.
template <typename TG>
cudaError_t launch_composite_bwd(const ViewParams& vp, const ForwardBuffers& fb, const float* bg, const float* dL_dpix,
                                 const float* dL_ddepth, const TG* dL_dfeat_pix, float dL_dfeat_pix_scale,
                                 float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dz,
                                 float* dL_dfeature, cudaStream_t s, const FeatureRows& feat = {},
                                 const float* dL_dalpha = nullptr, const float* dL_dinvdepth = nullptr);
// Feature lifting, R > 0: weight_sum[P] += the blend weights w = alpha*T of each Gaussian over the view and
// feature_sum[P, C] += sum_p w * map[:, p], through the same lists.  TF (float or __half) is the element type of map
template <typename TF>
cudaError_t launch_feature_lift(const ViewParams& vp, const ForwardBuffers& fb, const TF* map, float* feature_sum,
                                float* weight_sum, cudaStream_t s);
// Per-Gaussian scores, R > 0, from the same walk without lists or feature kernel: weight_sum[P] += sum_p w,
// max_weight[P] = max(max_weight, max_p w) (max_weight >= 0, compared as float bits), pixel_count[P] += the number of
// pixels the Gaussian blended into.  Allocates nothing
cudaError_t launch_gaussian_scores(const ViewParams& vp, const ForwardBuffers& fb, float* weight_sum, float* max_weight,
                                   int64_t* pixel_count, cudaStream_t s);

// ---- feature_head.cu (a float16 map or target gives the result of the float32 one upcast exactly; a float16 gradient
// is half_rn(out_scale * the float32 one), out_scale not read for a float gradient)
template <typename FM, typename GT>
cudaError_t launch_feature_resize_fwd(int C, int H, int W, int Hg, int Wg, const FM* fm, const GT* gt, float grad_scale,
                                      float* out, float* loss_sum, cudaStream_t s);
template <typename OUT>
cudaError_t launch_feature_resize_bwd(int C, int H, int W, int Hg, int Wg, const float* dout, OUT* dfm, float out_scale,
                                      cudaStream_t s);

// ---- image_loss.cu: fused L1 + SSIM sums and, with dL_dimage != nullptr, the gradient w.r.t. image
bool image_loss_grid_ok(int planes, int H, int W);  // the launch grid fits CUDA's limits
cudaError_t launch_image_loss(int planes, int H, int W, const float* image, const float* gt, float w_l1, float w_ssim,
                              float* sums, float* dL_dimage, cudaStream_t s);

// ---- feature_decoder.cu: 1x1-conv decoder y = W x + b, and its L1 loss with dL/dx (written), dL/dW and dL/db (added)
constexpr int kDecoderMaxCin = 256, kDecoderMaxCout = 4096;
bool decoder_grid_ok(int Cin, int Cout, int N);  // sizes in range and the launch grids fit CUDA's limits
// y may be float16 (rounded to nearest even, as torch's .half()); a float16 gt is upcast exactly
template <typename Y>
cudaError_t launch_decoder_forward(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x, Y* y,
                                   cudaStream_t s);
template <typename GT>
cudaError_t launch_decoder_l1(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                              const GT* gt, float grad_scale, float* loss_sum, float* dx, float* dW, float* db,
                              cudaStream_t s);
// W [Cout,Cin] -> wt [rows, Cp] rounded to TF32 and zero-padded; b [Cout] or NULL -> bp [rows] zero-padded
cudaError_t launch_decoder_prep(int Cin, int Cout, int Cp, int rows, const float* weight, const float* bias, float* wt,
                                float* bp, cudaStream_t s);

// ---- feature_query.cu: cosine similarity of (decoded) feature columns with text embeddings -> argmax label, softmax
// probability of a positive prompt set, logits.  weight == NULL: no decoder (D == C).  x may be float16 (upcast exactly)
constexpr int kQueryMaxK = 256, kQueryMaxD = 4096;
template <typename X>
cudaError_t launch_feature_query(int C, int D, int K, int N, const float* weight, const float* bias, const X* x,
                                 const float* text, float logit_scale, const uint8_t* positive, int64_t* labels,
                                 float* prob, float* logits, cudaStream_t s);

// ---- feature_pca.cu: PCA picture of a feature map x [C,N] (float16 x is upcast exactly).  scratch is
// pca_scratch_bytes(C, N) bytes, whose first pca_scratch_fixed_bytes(C, N) need no device query to size
constexpr int kPcaMinC = 3, kPcaMaxC = 1024;
cudaError_t pca_scratch_bytes(int C, int N, size_t* bytes);
size_t pca_scratch_fixed_bytes(int C, int N);
template <typename X>
cudaError_t launch_pca_moments(int C, int N, const X* x, char* scratch, float* mean, double* cov, cudaStream_t s);
template <typename X>
cudaError_t launch_pca_range(int C, int N, const X* x, const float* mean, const float* comp, char* scratch, float* range,
                             cudaStream_t s);
template <typename X>
cudaError_t launch_pca_image(int C, int N, const X* x, const float* mean, const float* comp, const float* range,
                             float* image, cudaStream_t s);

// ---- knn.cu: exact mean squared distance to the 3 nearest other points (distCUDA2); scratch is knn_scratch_bytes(P)
// bytes whose first knn_scratch_fixed_bytes(P) need no device query to size
cudaError_t knn_scratch_bytes(int P, size_t* bytes);
size_t knn_scratch_fixed_bytes(int P);
cudaError_t launch_knn_mean_dist(int P, const float* points, float* out, char* scratch, cudaStream_t s);

// ---- densify.cu: clone / split / prune (densify_and_prune) and reset_opacity.  scratch is densify_scratch_bytes(P)
// bytes whose first densify_scratch_fixed_bytes(P) (the scanned per-Gaussian flags apply reads) need no device query;
// src / dst are the 21 fields of f3dgs_gaussian_fields[3] in order
cudaError_t densify_scratch_bytes(int P, size_t* bytes);
size_t densify_scratch_fixed_bytes(int P);
cudaError_t launch_densify_plan(int P, const float* grad_accum, const float* denom, const float* raw_opacity,
                                const float* raw_scaling, float max_grad, float dense_scale, float min_opacity,
                                float max_world_scale, char* scratch, int32_t* counts, cudaStream_t s);
// prune from a mask: the plan of launch_densify_apply that keeps row i iff keep[i] != 0, counts {A, 0, 0, 0}
cudaError_t launch_prune_plan(int P, const uint8_t* keep, char* scratch, int32_t* counts, cudaStream_t s);
cudaError_t launch_densify_apply(int P, int M, int C, const char* scratch, const int32_t counts[4], const float* normals,
                                 const float* const src[21], float* const dst[21], cudaStream_t s);
cudaError_t launch_reset_opacity(int P, float* raw_opacity, float* exp_avg, float* exp_avg_sq, float ceiling,
                                 cudaStream_t s);

// ---- mcmc.cu: 3DGS-MCMC relocation, growth and position noise (include/f3dgs_b200.h: f3dgs_mcmc_*).  scratch is
// mcmc_scratch_bytes(P) bytes whose first mcmc_scratch_fixed_bytes(P) need no device query; fields are the 21 fields of
// f3dgs_gaussian_fields[3] in order
cudaError_t mcmc_scratch_bytes(int P, size_t* bytes);
size_t mcmc_scratch_fixed_bytes(int P);
cudaError_t launch_mcmc_plan(int P, const float* raw_opacity, float min_opacity, char* scratch, int32_t* n_dead,
                             int32_t* index, float* alive_opacity, cudaStream_t s);
cudaError_t launch_mcmc_relocate(int P, int M, int C, int n, const int32_t* dead, const int32_t* src, float min_opacity,
                                 float* const fields[21], __half* feature_f16, char* scratch, cudaStream_t s);
cudaError_t launch_mcmc_add(int P, int M, int C, int n, const int32_t* src, float min_opacity,
                            const float* const src_fields[21], float* const dst_fields[21], char* scratch,
                            cudaStream_t s);
cudaError_t launch_mcmc_inject_noise(int P, float* xyz, const float* raw_opacity, const float* raw_scaling,
                                     const float* raw_rotation, const float* eps, float scale, cudaStream_t s);

// ---- filter3d.cu: Mip-Splatting's 3D smoothing filter (include/f3dgs_b200.h: f3dgs_filter3d_*).  scratch is
// kFilter3dScratchBytes of device memory (the max seen depth)
constexpr size_t kFilter3dScratchBytes = 256;
cudaError_t launch_filter3d_compute(int P, int V, const float* means3D, const float* viewmatrices,
                                    const float* intrinsics, float* filter, int32_t* n_seen, char* scratch,
                                    cudaStream_t s);
cudaError_t launch_filter3d_apply(int P, const float* opacity, const float* scales, const float* filter,
                                  float* opacity_out, float* scales_out, cudaStream_t s);
cudaError_t launch_filter3d_apply_backward(int P, const float* opacity, const float* scales, const float* filter,
                                           const float* dL_dopacity_f, const float* dL_dscales_f, float* dL_dopacity,
                                           float* dL_dscales, cudaStream_t s);
cudaError_t launch_reset_opacity_filter3d(int P, float* raw_opacity, const float* raw_scaling, const float* filter,
                                          float* exp_avg, float* exp_avg_sq, float ceiling, cudaStream_t s);

// ---- optimizer.cu: activation prologue and fused Adam step (include/f3dgs_b200.h: f3dgs_activate / f3dgs_adam_step)
cudaError_t launch_activate(int P, int M, const float* raw_opacity, const float* raw_scaling, const float* raw_rotation,
                            const float* features_dc, const float* features_rest, float* opacity, float* scales,
                            float* rotations, float* shs, cudaStream_t s);
// param_f16 (IDENTITY only, may be NULL): also written, half_rn of the updated param.  visible (may be NULL): P bytes, the
// rows of n / P elements to update (nonzero); the others are left untouched.  step == 0: no bias correction
cudaError_t launch_adam_step(int kind, size_t n, int M, float* param, const float* grad_activated, float* exp_avg,
                             float* exp_avg_sq, float lr, float beta1, float beta2, float eps, int step, cudaStream_t s,
                             __half* param_f16 = nullptr, const uint8_t* visible = nullptr, int P = 0);

}  // namespace f3dgs
