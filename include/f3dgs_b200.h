/*
 * f3dgs_b200 -- C ABI of the H100-native feature-Gaussian rasterizer (libf3dgs_b200.so).
 *
 * This is the drop-in boundary below the Python/torch surface.  Every entry point takes plain
 * device pointers and sizes -- no torch, no C++ types -- and replaces one member of the
 * reference's inner C++ interface `CudaRasterizer::Rasterizer`
 * (reference: submodules/diff-gaussian-rasterization-feature/cuda_rasterizer/rasterizer.h:18-94).
 *
 *   reference                                     this library
 *   Rasterizer::forward      rasterizer.h:31-58   f3dgs_forward
 *   Rasterizer::backward     rasterizer.h:60-93   f3dgs_backward
 *   Rasterizer::markVisible  rasterizer.h:24-29   f3dgs_mark_visible
 *
 * Differences from the reference interface, all additive:
 *   - the feature width C (reference: compile-time NUM_SEMANTIC_CHANNELS, config.h:16) is a
 *     run-time argument, 0 <= C <= F3DGS_MAX_FEATURE_DIM;
 *   - the three std::function<char*(size_t)> allocators become (function pointer, context) pairs;
 *   - every call takes the CUDA stream to launch on (reference: legacy default stream);
 *   - errors are returned as negative codes with a message in f3dgs_last_error() instead of C++
 *     exceptions (reference: std::runtime_error from CHECK_CUDA, auxiliary.h:172-179).
 *
 * All float tensors are fp32 (except where a symbol's _f16 / _f16gt suffix says float16), contiguous, device
 * memory.  Matrices are the 16 floats of the
 * reference's row-major [4,4] torch tensors, i.e. column-major for the kernels
 * (auxiliary.h:58-77).  An absent optional input is a NULL pointer
 * (rasterize_points.cu: empty tensor -> nullptr).
 */
#ifndef F3DGS_B200_H_INCLUDED
#define F3DGS_B200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define F3DGS_ABI_VERSION 2
#define F3DGS_MAX_FEATURE_DIM 4096
#define F3DGS_TILE 16 /* BLOCK_X == BLOCK_Y == 16, reference config.h:18-19 */

/* error codes (returned negated) */
#define F3DGS_OK 0
#define F3DGS_ERR_INVALID_ARGUMENT 1
#define F3DGS_ERR_CUDA 2
#define F3DGS_ERR_ALLOC 3

/* Allocator callback: must return device memory of at least `bytes` bytes, 256-byte aligned,
 * valid until the matching backward call has finished (reference: the resize lambdas of
 * rasterize_points.cu:27-33).  Called exactly once per buffer per forward: geometry first,
 * image second, binning third (after the single host sync on num_rendered). */
typedef char* (*f3dgs_alloc_fn)(void* ctx, size_t bytes);

/* ---- forward: reference Rasterizer::forward, rasterizer_impl.cu:198-342 -------------------
 * Returns num_rendered (>= 0; number of (Gaussian, tile) instances) or -(error code).
 *   P            number of Gaussians           D  active SH degree (0..3)
 *   M            SH coefficients per colour in `shs` (0 if shs == NULL)
 *   C            feature width of semantic_feature / out_feature_map (run-time)
 *   background   [3]            means3D [P,3]        shs [P,M,3] or NULL
 *   colors_precomp [P,3] or NULL (exactly one of shs / colors_precomp)
 *   semantic_feature [P,C] (NULL iff C == 0)         opacities [P]
 *   scales [P,3] + rotations [P,4] (w,x,y,z), or cov3D_precomp [P,6]
 *   viewmatrix, projmatrix [16]  cam_pos [3]
 *   out_color [3,H,W]  out_feature_map [C,H,W]  out_depth [H,W]   (every element is written)
 *   radii [P] int32 (may be NULL: kept internally)
 *   debug != 0: synchronise and check after every stage (reference CHECK_CUDA semantics)
 */
int f3dgs_forward(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx,
                  f3dgs_alloc_fn binning_alloc, void* binning_ctx,
                  f3dgs_alloc_fn image_alloc, void* image_ctx,
                  int P, int D, int M, int C,
                  const float* background, int width, int height,
                  const float* means3D, const float* shs, const float* colors_precomp,
                  const float* semantic_feature, const float* opacities,
                  const float* scales, float scale_modifier, const float* rotations,
                  const float* cov3D_precomp,
                  const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                  float tan_fovx, float tan_fovy, int prefiltered,
                  float* out_color, float* out_feature_map, float* out_depth, int* radii,
                  int debug, void* cuda_stream);

/* ---- backward: reference Rasterizer::backward, rasterizer_impl.cu:347-461 -----------------
 * R is the num_rendered returned by the matching forward; the three buffers are the ones the
 * allocators returned.  All dL_d* outputs must be ZERO-FILLED by the caller (the reference
 * wrapper allocates them with torch::zeros, rasterize_points.cu:163-173); gradients are
 * accumulated into them.  dL_dconic [P,4] and dL_dz [P] are scratch outputs like in the
 * reference.  Returns 0 or -(error code).
 */
int f3dgs_backward(int P, int D, int M, int R, int C,
                   const float* background, int width, int height,
                   const float* means3D, const float* shs, const float* colors_precomp,
                   const float* semantic_feature,
                   const float* scales, float scale_modifier, const float* rotations,
                   const float* cov3D_precomp,
                   const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                   float tan_fovx, float tan_fovy, const int* radii,
                   char* geom_buffer, char* binning_buffer, char* image_buffer,
                   const float* dL_dpix, const float* dL_dfeaturepix, const float* dL_depths,
                   float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                   float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                   float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz,
                   int debug, void* cuda_stream);

/* ---- accumulating backward for view batches (additive: the reference ASSIGNS per-view gradients into freshly
 * zero-filled tensors, rasterize_points.cu:163-173, backward.cu:273, and leaves the sum over views to autograd) ----
 * Same inputs as f3dgs_backward.  Differences:
 *   - every per-parameter gradient (dL_dopacity [P], dL_dsemantic_feature [P,C], dL_dmean3D [P,3], dL_dsh [P,M,3],
 *     dL_dscale [P,3], dL_drot [P,4], and dL_dcolors_precomp [P,3] / dL_dcov3D_precomp [P,6] when those are the inputs,
 *     NULL otherwise) is ACCUMULATED (+=): the caller zeroes them once per step, e.g. as slices of one flat buffer that
 *     is then all-reduced once;
 *   - the per-view intermediates (screen-space mean, conic, depth, colour and covariance gradients) live in `scratch`
 *     (f3dgs_backward_scratch_bytes(P) bytes of device memory, 256-byte aligned), which the call zeroes itself;
 *   - dL_dmean2D_out (optional, [P,3]) receives this view's screen-space gradient (the reference's
 *     viewspace_point_tensor.grad);
 *   - grad_accum / denom (optional, both or neither, [P]): the densification statistics of the reference training loop
 *     (scene/gaussian_model.py:436-438): for radii > 0, grad_accum += ||dL_dmean2D.xy||, denom += 1;
 *   - composite_done_event (optional cudaEvent_t): recorded on the stream after the backward composite kernel, i.e. when
 *     dL_dsemantic_feature and dL_dopacity of this view are complete (the backward preprocess does not touch them), so
 *     that a collective on that bucket can start on another stream while the preprocess still runs.
 */
size_t f3dgs_backward_scratch_bytes(int P);
int f3dgs_backward_accum(int P, int D, int M, int R, int C,
                         const float* background, int width, int height,
                         const float* means3D, const float* shs, const float* colors_precomp,
                         const float* scales, float scale_modifier, const float* rotations,
                         const float* cov3D_precomp,
                         const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                         float tan_fovx, float tan_fovy, const int* radii,
                         char* geom_buffer, char* binning_buffer, char* image_buffer,
                         const float* dL_dpix, const float* dL_dfeaturepix, const float* dL_depths,
                         char* scratch,
                         float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature,
                         float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale,
                         float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                         void* composite_done_event, int debug, void* cuda_stream);

/* ==== callers either side of the rasterizer (SURVEY.md section 8 f): additive entry points ======================= */

/* ---- post-raster feature head: reference train.py:98-104 ---------------------------------------------------------
 * F.interpolate(feature_map[C,H,W] -> [C,Hg,Wg], mode='bilinear', align_corners=True) fused with l1_loss against the
 * teacher map and its gradient.
 *   f3dgs_feature_resize_fwd  gt != NULL: out[C,Hg,Wg] = sign(resized - gt) * grad_scale  (dL/d resized for
 *                             L = grad_scale * sum |resized - gt|; pass weight / (C*Hg*Wg) for the weighted mean) and
 *                             *loss_sum += sum |resized - gt|  (device float, caller-zeroed, may be NULL);
 *                             gt == NULL: out = resized map (decoder path: f3dgs_decoder_l1 below runs the
 *                             1x1 convolution of models/networks.py:107-119 and its loss between the two calls).
 *   f3dgs_feature_resize_bwd  dL_dfeature_map[C,H,W] = resize^T(dout[C,Hg,Wg]); every element is written (gather, no
 *                             atomics, no zero fill needed).
 */
int f3dgs_feature_resize_fwd(int C, int H, int W, int Hg, int Wg, const float* feature_map, const float* gt,
                             float grad_scale, float* out, float* loss_sum, void* cuda_stream);
int f3dgs_feature_resize_bwd(int C, int H, int W, int Hg, int Wg, const float* dout, float* dL_dfeature_map,
                             void* cuda_stream);
/* f3dgs_feature_resize_fwd with a float16 teacher map (the data format's <name>_fmap_CxHxW.pt): gt [C,Hg,Wg] holds IEEE
 * binary16 bits and is required.  The result is that of f3dgs_feature_resize_fwd applied to the exactly upcast float32
 * target.  It validates as its float32 twin does, and also rejects an `out` that overlaps feature_map or gt. */
int f3dgs_feature_resize_fwd_f16gt(int C, int H, int W, int Hg, int Wg, const float* feature_map, const uint16_t* gt,
                                   float grad_scale, float* out, float* loss_sum, void* cuda_stream);

/* ---- feature decoder (--speedup): models/networks.py:107-119 CNN_decoder, nn.Conv2d(Cin, Cout, kernel_size=1) -------
 * x [Cin,N] (the resized map, N = Hg*Wg), weight [Cout,Cin] (the conv weight [Cout,Cin,1,1] as contiguous memory),
 * bias [Cout] or NULL (a conv without bias), gt [Cout,N].  1 <= Cin <= 256, 1 <= Cout <= 4096, N >= 1.  TF32 tensor-core
 * products (operands rounded to nearest, fp32 accumulate), the precision of cuDNN's default for the reference layer.
 *   f3dgs_decoder_forward  y[Cout,N] = weight x + bias; y must not overlap an input.
 *   f3dgs_decoder_l1       with s = sign(y - gt) (sign(0) = 0):  *loss_sum = sum |y - gt| (written);
 *                          dL_dx[Cin,N] = grad_scale * weight^T s (every element written; must not overlap an input);
 *                          dL_dweight[Cout,Cin] += grad_scale * s x^T;  dL_dbias[Cout] += grad_scale * sum_n s
 *                          (added, so that the views of a step accumulate; dL_dbias may be NULL iff bias is NULL).
 *                          l1_loss(decoder(x), gt) * w takes grad_scale = w / (Cout * N).
 * y and s never reach memory as fp32; results are bitwise reproducible (no float atomics). */
int f3dgs_decoder_forward(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x, float* y,
                          void* cuda_stream);
int f3dgs_decoder_l1(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x, const float* gt,
                     float grad_scale, float* loss_sum, float* dL_dx, float* dL_dweight, float* dL_dbias,
                     void* cuda_stream);
/* float16 variants; half data is IEEE binary16 bits in uint16_t, and overlap checks use its 2-byte size.
 *   f3dgs_decoder_l1_f16gt    gt [Cout,N] float16.  The result is that of f3dgs_decoder_l1 applied to the exactly upcast
 *                             float32 target (bitwise, like the float32 call itself).  Validates as f3dgs_decoder_l1.
 *   f3dgs_decoder_forward_f16 y [Cout,N] float16: the y of f3dgs_decoder_forward rounded to nearest even (torch's
 *                             .half(): +-inf beyond 65504).  Validates as f3dgs_decoder_forward. */
int f3dgs_decoder_l1_f16gt(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                           const uint16_t* gt, float grad_scale, float* loss_sum, float* dL_dx, float* dL_dweight,
                           float* dL_dbias, void* cuda_stream);
int f3dgs_decoder_forward_f16(int Cin, int Cout, int N, const float* weight, const float* bias, const float* x,
                              uint16_t* y, void* cuda_stream);

/* ---- photometric loss: reference train.py (colour term), utils/loss_utils.py l1_loss + ssim(window_size=11) ---------
 * loss = (1 - lambda_dssim) * l1_loss(image, gt) + lambda_dssim * (1 - ssim(image, gt)).  image, gt [planes,H,W]; the
 * SSIM window is the 11-tap Gaussian (sigma 1.5) per plane with zero padding, C1 = 0.01^2, C2 = 0.03^2.
 *   sums       device float[2]: sum |image - gt|, sum of the SSIM map (WRITTEN, not accumulated)
 *   dL_dimage  [planes,H,W] or NULL (value only): w_l1 * sign(image - gt) + w_ssim * d(sum ssim_map)/d image, every
 *              element written; must not overlap image or gt.  The reference loss takes w_l1 = (1 - lambda) / N and
 *              w_ssim = -lambda / N with N = planes * H * W.
 * Deterministic: the same inputs give bitwise-identical sums and gradient.  planes == 0 is a no-op. */
int f3dgs_image_loss(int planes, int H, int W, const float* image, const float* gt, float w_l1, float w_ssim,
                     float* sums, float* dL_dimage, void* cuda_stream);

/* ---- activation prologue: reference scene/gaussian_model.py:98-121 ------------------------------------------------
 * opacity = sigmoid(raw_opacity[P]); scales = exp(raw_scaling[P,3]); rotations = normalize(raw_rotation[P,4]);
 * shs[P,M,3] = cat(features_dc[P,1,3], features_rest[P,M-1,3]).  Any raw pointer may be NULL (group skipped). */
int f3dgs_activate(int P, int M, const float* raw_opacity, const float* raw_scaling, const float* raw_rotation,
                   const float* features_dc, const float* features_rest, float* opacity, float* scales,
                   float* rotations, float* shs, void* cuda_stream);

/* ---- fused optimizer step: reference scene/gaussian_model.py:163-190 (torch.optim.Adam, one call per group) --------
 * `grad_activated` is the gradient w.r.t. the ACTIVATED tensor as the rasterizer's backward produces it; `kind` names
 * the activation whose Jacobian is applied before the Adam update of the raw parameter (n elements, in place):
 *   IDENTITY (xyz, semantic features)   SIGMOID (opacity)   EXP (scaling)   NORMALIZE4 (rotation, n % 4 == 0)
 *   SH_DC / SH_REST: the raw parameter is features_dc [P,1,3] / features_rest [P,M-1,3], the gradient the [P,M,3] SH tensor.
 * step >= 1 is the 1-based Adam step count of the group (bias correction). */
#define F3DGS_PARAM_IDENTITY 0
#define F3DGS_PARAM_SIGMOID 1
#define F3DGS_PARAM_EXP 2
#define F3DGS_PARAM_NORMALIZE4 3
#define F3DGS_PARAM_SH_DC 4
#define F3DGS_PARAM_SH_REST 5
int f3dgs_adam_step(int kind, size_t n, int M, float* param, const float* grad_activated, float* exp_avg,
                    float* exp_avg_sq, float lr, float beta1, float beta2, float eps, int step, void* cuda_stream);

/* ---- initial scales: reference submodules/simple-knn distCUDA2, used by scene/gaussian_model.py:133-160 ------------
 * out[i] = (d0 + d1 + d2) / 3 in fp32, where d0 <= d1 <= d2 are the three smallest squared distances from points[i] to
 * the points j != i (exclusion by index: a coincident point counts as 0).  Missing neighbours (P < 4) keep FLT_MAX, as in
 * the reference: +inf for P = 1, 2 and about FLT_MAX / 3 for P = 3.  The result is exact (not approximate), bitwise
 * reproducible and independent of the order of the points.
 *   points   [P,3] float32 device memory        out  [P] float32, must not overlap points or scratch
 *   scratch  f3dgs_knn_scratch_bytes(P) bytes of device memory, 256-byte aligned
 * Stream-ordered with no host sync.  P == 0 launches nothing.  f3dgs_knn_scratch_bytes returns 0 for P <= 0, and 0 with
 * f3dgs_last_error() set if the size query of the device sort fails. */
size_t f3dgs_knn_scratch_bytes(int P);
int f3dgs_knn_mean_dist(int P, const float* points, float* out, char* scratch, void* cuda_stream);

/* ---- adaptive density control: reference scene/gaussian_model.py:350-434 (densify_and_prune: clone :407-418,
 * split :381-405, prune :316-330) and :231-234 (reset_opacity) ----------------------------------------------------
 * The seven raw parameter fields of P Gaussians (f_rest is NULL when M == 1, semantic_feature NULL when C == 0):
 *   xyz [P,3]  f_dc [P,1,3]  f_rest [P,M-1,3]  opacity [P,1]  scaling [P,3] (log)  rotation [P,4]  semantic_feature [P,1,C]
 * Densification is two calls with one host read in between:
 *   f3dgs_densify_plan   classifies every Gaussian and writes counts = {A, B, Cc, Ns} (device int32[4]): A originals
 *                        kept, B clones kept, Cc children kept per split copy, Ns Gaussians selected for split.  With
 *                        g = grad_accum / denom (0 where NaN) and smax = max of expf(raw_scaling) over 3, in fp32:
 *                          clone  g >= max_grad && smax <= dense_scale     (dense_scale = percent_dense * extent)
 *                          split  g >= max_grad && smax >  dense_scale
 *                          prune  sigmoid(opacity) < min_opacity || smax > max_world_scale (0.1 * extent; +inf
 *                                 disables it), each row on its own scaling
 *                        The thresholds are the caller's doubles rounded once to float, as torch compares.
 *   f3dgs_densify_apply  writes the P' = A + B + 2 Cc output rows: the order-preserving compaction of
 *                        [P originals | clones | split copy 0 | split copy 1] without the split originals and the
 *                        pruned rows.  Every field of a clone or child is its parent's, except a child's
 *                        scaling = logf(expf(s) * (1 / 1.6f)) and xyz = R(q) (z * expf(s)) + parent xyz, with
 *                        R(q) of q = r / sqrt(sum r^2) and z = normals[Ns * copy + (split index), :].
 *                        src[0] / dst[0] are the raw fields, [1] exp_avg, [2] exp_avg_sq: kept rows move their
 *                        moments bitwise, clone and child rows get zeros.  counts is the HOST copy of what plan wrote
 *                        (it sizes dst and normals [2 Ns, 3]); if it differs from the device counts nothing is
 *                        written.  No dst field may overlap a src field, normals or the scratch.
 *   scratch  f3dgs_densify_scratch_bytes(P) bytes of device memory, 256-byte aligned, unchanged between the calls
 * Both calls are stream-ordered without host sync and bitwise deterministic.  3 P must not exceed INT_MAX.
 * f3dgs_densify_scratch_bytes returns 0 for P <= 0, and 0 with f3dgs_last_error() set if the size query fails.
 *
 * f3dgs_reset_opacity: raw_opacity <- logf(x / (1 - x)) with x = min(sigmoid(raw_opacity), ceiling) (NaN propagates, as
 * torch.minimum), in place; exp_avg and exp_avg_sq of the opacity [P] are zeroed.  The reference's ceiling is 0.01f. */
typedef struct f3dgs_gaussian_fields {
    float *xyz, *f_dc, *f_rest, *opacity, *scaling, *rotation, *semantic_feature;
} f3dgs_gaussian_fields;
size_t f3dgs_densify_scratch_bytes(int P);
int f3dgs_densify_plan(int P, const float* grad_accum, const float* denom, const float* raw_opacity,
                       const float* raw_scaling, float max_grad, float dense_scale, float min_opacity,
                       float max_world_scale, char* scratch, int32_t* counts, void* cuda_stream);
int f3dgs_densify_apply(int P, int M, int C, const char* scratch, const int32_t counts[4], const float* normals,
                        const f3dgs_gaussian_fields src[3], const f3dgs_gaussian_fields dst[3], void* cuda_stream);
int f3dgs_reset_opacity(int P, float* raw_opacity, float* exp_avg, float* exp_avg_sq, float ceiling, void* cuda_stream);

/* ---- markVisible: reference rasterizer_impl.cu:141-153 (checkFrustum :54-66) --------------
 * present[i] = (view-space z of means3D[i] > 0.2).  `present` is P bytes (0/1). */
int f3dgs_mark_visible(int P, const float* means3D, const float* viewmatrix,
                       const float* projmatrix, uint8_t* present, void* cuda_stream);

/* ---- introspection for the parity harness --------------------------------------------------
 * Byte offsets of the fields inside the three opaque buffers (the layout is private to this
 * library; the reference's is rasterizer_impl.cu:154-194).  Offsets are relative to the
 * 256-byte-aligned base pointer the allocator returned.
 */
typedef struct f3dgs_layout {
    /* geometry buffer (P entries) */
    size_t geom_bytes;
    size_t geom_rec;        /* float4[3P]: {x,y,ext_x,ext_y} {conic a,b,c,opacity} {r,g,b,depth} */
    size_t geom_cov3d;      /* float[6P] */
    size_t geom_clamped;    /* uint8[P]  bit k set = colour channel k was clamped at 0 */
    size_t geom_tiles;      /* uint32[P] tiles touched */
    size_t geom_offsets;    /* uint32[P] inclusive scan of tiles touched */
    size_t geom_radii;      /* int32[P]  internal radii */
    /* image buffer */
    size_t img_bytes;
    size_t img_final_T;     /* float[H*W] */
    size_t img_n_contrib;   /* uint32[H*W] */
    size_t img_ranges;      /* uint2[tiles] */
    /* binning buffer (R entries) */
    size_t bin_bytes;
    size_t bin_point_list;  /* uint32[R] sorted Gaussian ids */
    size_t bin_keys;        /* uint64[R] sorted keys */
} f3dgs_layout;

int f3dgs_get_layout(int P, int width, int height, int R, f3dgs_layout* out);

/* Number of this library's own kernels launched in this process (CUB's scan/sort kernels are not
 * counted) -- bench.py reports the delta over its timed region as gpu_launches. */
unsigned long long f3dgs_launch_count(void);

/* ---- per-stage device timing (bench.py roofline) ---------------------------------------------
 * When enabled, every stage is bracketed by CUDA events on the launch stream (no host sync).
 * f3dgs_profile_read synchronises the recorded events, adds the elapsed milliseconds and launch
 * counts per stage into ms[F3DGS_N_STAGES] / count[F3DGS_N_STAGES] and clears the recordings.
 * Stage ids: */
#define F3DGS_STAGE_PREPROCESS_FWD 0
#define F3DGS_STAGE_SCAN 1
#define F3DGS_STAGE_DUPLICATE_KEYS 2
#define F3DGS_STAGE_SORT 3
#define F3DGS_STAGE_TILE_RANGES 4
#define F3DGS_STAGE_COMPOSITE_FWD 5
#define F3DGS_STAGE_COMPOSITE_BWD 6
#define F3DGS_STAGE_PREPROCESS_BWD 7
#define F3DGS_N_STAGES 8
void f3dgs_profile_enable(int on);
int f3dgs_profile_read(double* ms, unsigned long long* count);

/* Last error message of the calling thread ("" if none). */
const char* f3dgs_last_error(void);

int f3dgs_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* F3DGS_B200_H_INCLUDED */
