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
#define F3DGS_CAMERA_GRAD_FLOATS 35 /* dL_dcamera of the _cam backward entries */
/* element-type codes of the _feature_geometry, _antialiased and _alpha_invdepth entries */
#define F3DGS_F32 0 /* IEEE binary32 */
#define F3DGS_F16 1 /* IEEE binary16 */

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
/* f3dgs_forward with float16 features (rendering a trained field): semantic_feature [P,C] and out_feature_map [C,H,W]
 * hold IEEE binary16 bits; every other argument is as above.  The feature map is bitwise that of f3dgs_forward for the
 * exactly upcast features, rounded once to nearest even (torch's .half()); colour, depth, radii, num_rendered and the
 * three buffers are bitwise those of f3dgs_forward, so f3dgs_backward takes them as they are (it does not read the
 * features).  Validates as f3dgs_forward. */
int f3dgs_forward_f16(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx,
                      f3dgs_alloc_fn binning_alloc, void* binning_ctx,
                      f3dgs_alloc_fn image_alloc, void* image_ctx,
                      int P, int D, int M, int C,
                      const float* background, int width, int height,
                      const float* means3D, const float* shs, const float* colors_precomp,
                      const uint16_t* semantic_feature, const float* opacities,
                      const float* scales, float scale_modifier, const float* rotations,
                      const float* cov3D_precomp,
                      const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                      float tan_fovx, float tan_fovy, int prefiltered,
                      float* out_color, uint16_t* out_feature_map, float* out_depth, int* radii,
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
/* f3dgs_backward with a float16 feature-map gradient (training float16 feature fields): dL_dfeaturepix [C,H,W] holds
 * IEEE binary16 bits h standing for the gradient dL_dfeaturepix_scale * float(h) (finite, nonzero).  The scale lets a
 * gradient far below float16's range (an L1 feature loss's weight / (C*Hg*Wg) is ~1e-8) be stored without underflow;
 * it is applied in float32 (one multiply, rounded to nearest) as the map is loaded, and no float32 [C,H,W] buffer is
 * made.  Every output equals that of f3dgs_backward called with the float32 map scale * float(h), up to the order of
 * the float reductions f3dgs_backward already has; dL_dsemantic_feature stays float32 (the master gradient) and must
 * not overlap dL_dfeaturepix.  Validates as f3dgs_backward. */
int f3dgs_backward_f16(int P, int D, int M, int R, int C,
                       const float* background, int width, int height,
                       const float* means3D, const float* shs, const float* colors_precomp,
                       const float* semantic_feature,
                       const float* scales, float scale_modifier, const float* rotations,
                       const float* cov3D_precomp,
                       const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                       float tan_fovx, float tan_fovy, const int* radii,
                       char* geom_buffer, char* binning_buffer, char* image_buffer,
                       const float* dL_dpix, const uint16_t* dL_dfeaturepix, float dL_dfeaturepix_scale,
                       const float* dL_depths,
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
 *     that a collective on that bucket can start on another stream while the preprocess still runs.  In the
 *     antialiased entry (below) the preprocess finishes dL_dopacity, so the event is recorded after it.
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
/* f3dgs_backward_accum with a float16 feature-map gradient, scaled as for f3dgs_backward_f16.  Arguments are validated
 * before the scratch is zeroed. */
int f3dgs_backward_accum_f16(int P, int D, int M, int R, int C,
                             const float* background, int width, int height,
                             const float* means3D, const float* shs, const float* colors_precomp,
                             const float* scales, float scale_modifier, const float* rotations,
                             const float* cov3D_precomp,
                             const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                             float tan_fovx, float tan_fovy, const int* radii,
                             char* geom_buffer, char* binning_buffer, char* image_buffer,
                             const float* dL_dpix, const uint16_t* dL_dfeaturepix, float dL_dfeaturepix_scale,
                             const float* dL_depths, char* scratch,
                             float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature,
                             float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale,
                             float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                             void* composite_done_event, int debug, void* cuda_stream);

/* ---- camera gradients (pose refinement, localisation, tracking): the _cam twins of the four backward entries ----
 * Each takes its twin's arguments plus a final dL_dcamera of F3DGS_CAMERA_GRAD_FLOATS (35) floats of device memory and
 * ADDS (+=) this view's camera gradient to it; every other output is bitwise its twin's.  Layout:
 *   [0, 16)   dL/dviewmatrix, [16, 32) dL/dprojmatrix: in the 16-float layout of the input matrices;
 *   [32, 35)  dL/dcampos.
 * The entries the forward never reads (viewmatrix[3,7,11,15], projmatrix[2,6,10,14]) get 0, and dL/dcampos gets only
 * the SH view-direction term (0 with colors_precomp).  A clamped view-space coordinate of the EWA Jacobian passes no
 * gradient, as for dL_dmean3D.  The feature map does not feed the geometry (SURVEY D.1): a loss on features alone gives
 * a zero camera gradient, as it gives a zero dL_dmean3D (the _feature_geometry entries below lift that).
 * The sum over Gaussians is free of floating-point atomics: float32 per-Gaussian terms, float64 block partials (taken
 * from the device's default memory pool; F3DGS_ERR_ALLOC if that fails) reduced in a fixed order, then rounded once and
 * added, so equal inputs give bitwise-equal results.  A NULL dL_dcamera, or one that overlaps another output (or the
 * scratch of the accumulating entries), is F3DGS_ERR_INVALID_ARGUMENT; P == 0 leaves it untouched. */
int f3dgs_backward_cam(int P, int D, int M, int R, int C,
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
                       int debug, void* cuda_stream, float* dL_dcamera);
int f3dgs_backward_cam_f16(int P, int D, int M, int R, int C,
                           const float* background, int width, int height,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* semantic_feature,
                           const float* scales, float scale_modifier, const float* rotations,
                           const float* cov3D_precomp,
                           const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                           float tan_fovx, float tan_fovy, const int* radii,
                           char* geom_buffer, char* binning_buffer, char* image_buffer,
                           const float* dL_dpix, const uint16_t* dL_dfeaturepix, float dL_dfeaturepix_scale,
                           const float* dL_depths,
                           float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                           float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                           float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz,
                           int debug, void* cuda_stream, float* dL_dcamera);
int f3dgs_backward_accum_cam(int P, int D, int M, int R, int C,
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
                             void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera);
int f3dgs_backward_accum_cam_f16(int P, int D, int M, int R, int C,
                                 const float* background, int width, int height,
                                 const float* means3D, const float* shs, const float* colors_precomp,
                                 const float* scales, float scale_modifier, const float* rotations,
                                 const float* cov3D_precomp,
                                 const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                 float tan_fovx, float tan_fovy, const int* radii,
                                 char* geom_buffer, char* binning_buffer, char* image_buffer,
                                 const float* dL_dpix, const uint16_t* dL_dfeaturepix, float dL_dfeaturepix_scale,
                                 const float* dL_depths, char* scratch,
                                 float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature,
                                 float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale,
                                 float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                                 void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera);

/* ---- feature gradients into geometry (opt-in; no reference counterpart: the reference disables the line,
 * backward.cu:575, and every other backward entry here keeps that, SURVEY D.1) ----
 * f3dgs_backward_feature_geometry takes f3dgs_backward's arguments and f3dgs_backward_accum_feature_geometry those of
 * f3dgs_backward_accum, with contracts unchanged, except that:
 *   - semantic_feature [P,C] (the forward's features) is read, of element type semantic_feature_dtype (F3DGS_F32, or
 *     F3DGS_F16 upcast exactly, as the forward reads it);
 *   - dL_dfeaturepix [C,H,W] has element type dL_dfeaturepix_dtype: F3DGS_F32, or F3DGS_F16 standing for
 *     dL_dfeaturepix_scale * float(h) as in f3dgs_backward_f16 (the scale is not read for F3DGS_F32);
 *   - dL_dcamera (optional, NULL: none) is the _cam entries' 35-float camera gradient, added to;
 *   - the feature map's gradient also feeds dL/dalpha, so that it reaches dL_dopacity, the screen-space mean and conic
 *     and, through them, dL_dmean3D, dL_dscale, dL_drot, dL_dcov3D and dL_dcamera.  For pixel p with blend weights
 *     w_i = alpha_i T_i (front to back) and d_ip = f_i . dL_dfeaturepix[:,p] (a C-wide dot product), the term added is
 *         dL/dalpha_i += T_i (d_ip - A_i),   A_i = alpha_{i+1} d_{i+1,p} + (1 - alpha_{i+1}) A_{i+1},   A_last = 0,
 *     the colour channels' recurrence with one channel d and a zero feature background (the feature map has none).
 * dL_dsemantic_feature, dL_dcolor and dL_dz are bitwise those of the counterpart; with a zero dL_dfeaturepix every output
 * is.  The densification statistics (grad_accum += ||dL_dmean2D.xy||) and dL_dmean2D_out include the feature term.  The
 * term costs two more kernels over the backward's per-block instance lists.  With C == 0 these entries are their
 * counterparts.  F3DGS_ERR_INVALID_ARGUMENT, before any launch, for a NULL semantic_feature with C > 0, an unknown dtype
 * code, a float16 map's scale that is not finite and nonzero, semantic_feature overlapping an output, and whatever the
 * counterpart (or, with dL_dcamera, its _cam twin) rejects. */
int f3dgs_backward_feature_geometry(int P, int D, int M, int R, int C,
                                    const float* background, int width, int height,
                                    const float* means3D, const float* shs, const float* colors_precomp,
                                    const void* semantic_feature, int semantic_feature_dtype,
                                    const float* scales, float scale_modifier, const float* rotations,
                                    const float* cov3D_precomp,
                                    const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                    float tan_fovx, float tan_fovy, const int* radii,
                                    char* geom_buffer, char* binning_buffer, char* image_buffer,
                                    const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                                    float dL_dfeaturepix_scale, const float* dL_depths,
                                    float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                                    float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                                    float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz,
                                    int debug, void* cuda_stream, float* dL_dcamera);
int f3dgs_backward_accum_feature_geometry(int P, int D, int M, int R, int C,
                                          const float* background, int width, int height,
                                          const float* means3D, const float* shs, const float* colors_precomp,
                                          const void* semantic_feature, int semantic_feature_dtype,
                                          const float* scales, float scale_modifier, const float* rotations,
                                          const float* cov3D_precomp,
                                          const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                          float tan_fovx, float tan_fovy, const int* radii,
                                          char* geom_buffer, char* binning_buffer, char* image_buffer,
                                          const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                                          float dL_dfeaturepix_scale, const float* dL_depths, char* scratch,
                                          float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature,
                                          float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale,
                                          float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                                          void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera);

/* ---- antialiased rendering (opt-in; no reference counterpart: the reference dilates every 2-D covariance by 0.3 px^2
 * and keeps the opacity, SURVEY A.2 step 5) ----
 * The dilation is a low-pass filter that does not conserve energy: a Gaussian at or below a pixel on screen is widened
 * but keeps its full opacity, so it is too thick and too bright, the more so the lower the rendering resolution.  The
 * antialiased forward multiplies the opacity by the ratio of the undilated to the dilated splat's integral:
 *     det0 = a0 c0 - b^2 (2-D covariance S = T V T^T before the dilation),  det = (a0 + 0.3)(c0 + 0.3) - b^2,
 *     rho = sqrt(max(2.5e-5, det0 / det)),   op_eff = opacity * rho,
 * and blends op_eff: it is the op of the splat records.  Conic, radii, tiles, depth, colour and everything else are those
 * of the default forward; the render is bitwise the default forward's with opacities := op_eff.
 *   f3dgs_forward_antialiased: f3dgs_forward's arguments, except that semantic_feature [P,C] and out_feature_map [C,H,W]
 *     are of element type semantic_feature_dtype (F3DGS_F32, or F3DGS_F16 as f3dgs_forward_f16).
 *   f3dgs_backward_antialiased / f3dgs_backward_accum_antialiased: the arguments and contracts of
 *     f3dgs_backward_feature_geometry / f3dgs_backward_accum_feature_geometry, except that semantic_feature may be NULL
 *     (no feature term: the counterpart without the feature term); dL_dcamera stays optional.  The composite's opacity
 *     gradient g = dL/dop_eff becomes dL_dopacity = rho g, and rho's dependence on (a, b, c) joins the conic's gradient:
 *         h = op_eff g / 2 (0 where rho is clamped),  dL/da += h (c0/det0 - c/det),  dL/dc += h (a0/det0 - a/det),
 *         dL/db += 2 h b (1/det - 1/det0),
 *     which reaches dL_dmean3D, dL_dscale, dL_drot, dL_dcov3D and dL_dcamera.  Where rho is clamped (a degenerate
 *     undilated covariance among those: det0 = 0) it is constant and only dL_dopacity = rho g is added.  With dL_dcamera
 *     every other output is bitwise that of the call without it, and one view accumulated into zeros gives the
 *     assigning entry's bits, as for the default entries.  dL_dmean2D, dL_dconic, dL_dcolor,
 *     dL_dsemantic_feature and dL_dz are the composite's, bitwise those of the counterpart on a forward with
 *     opacities := op_eff.  The assigning entry lets the composite write g into the zero-filled dL_dopacity and rescales
 *     it in place; the accumulating entry takes P floats for g from the device's default memory pool (F3DGS_ERR_ALLOC
 *     if that fails) and adds rho g into dL_dopacity.  f3dgs_backward_scratch_bytes is unchanged.
 *     composite_done_event is recorded after the backward preprocess, not the composite: only then is dL_dopacity final.
 *     F3DGS_ERR_INVALID_ARGUMENT, before any launch, for an unknown dtype code, dL_dopacity overlapping another output
 *     and whatever the counterpart rejects.
 * Contract (not checkable without a host sync, like R): the buffers of an antialiased forward go to the antialiased
 * backwards, or to f3dgs_lift_features_accum[_f16], and those of any other forward to the other backwards.  A mismatch
 * gives wrong gradients, not an error. */
int f3dgs_forward_antialiased(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx,
                              f3dgs_alloc_fn binning_alloc, void* binning_ctx,
                              f3dgs_alloc_fn image_alloc, void* image_ctx,
                              int P, int D, int M, int C,
                              const float* background, int width, int height,
                              const float* means3D, const float* shs, const float* colors_precomp,
                              const void* semantic_feature, int semantic_feature_dtype, const float* opacities,
                              const float* scales, float scale_modifier, const float* rotations,
                              const float* cov3D_precomp,
                              const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                              float tan_fovx, float tan_fovy, int prefiltered,
                              float* out_color, void* out_feature_map, float* out_depth, int* radii,
                              int debug, void* cuda_stream);
int f3dgs_backward_antialiased(int P, int D, int M, int R, int C,
                               const float* background, int width, int height,
                               const float* means3D, const float* shs, const float* colors_precomp,
                               const void* semantic_feature, int semantic_feature_dtype,
                               const float* scales, float scale_modifier, const float* rotations,
                               const float* cov3D_precomp,
                               const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                               float tan_fovx, float tan_fovy, const int* radii,
                               char* geom_buffer, char* binning_buffer, char* image_buffer,
                               const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                               float dL_dfeaturepix_scale, const float* dL_depths,
                               float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                               float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                               float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz,
                               int debug, void* cuda_stream, float* dL_dcamera);
int f3dgs_backward_accum_antialiased(int P, int D, int M, int R, int C,
                                     const float* background, int width, int height,
                                     const float* means3D, const float* shs, const float* colors_precomp,
                                     const void* semantic_feature, int semantic_feature_dtype,
                                     const float* scales, float scale_modifier, const float* rotations,
                                     const float* cov3D_precomp,
                                     const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                     float tan_fovx, float tan_fovy, const int* radii,
                                     char* geom_buffer, char* binning_buffer, char* image_buffer,
                                     const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                                     float dL_dfeaturepix_scale, const float* dL_depths, char* scratch,
                                     float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature,
                                     float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale,
                                     float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                                     void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera);

/* ---- opacity and inverse-depth maps (opt-in; no reference counterpart: the upstream 3DGS rasterizer's 2024 update
 * returns an inverse-depth map, and its image buffer's final transmittance is the opacity map's complement) ----
 * For pixel p the composite blends pairs i front to back with w_i = alpha_i T_i, exactly as the other forwards do.  The
 * _alpha_invdepth entries add two float32 planes [1,H,W] (whatever the feature element type):
 *     alpha     A_p = 1 - T_final,p       written as 1.f - T from the T that goes to final_T: bitwise 1 - final_T;
 *     invdepth  I_p = sum_i w_i / z_i     z_i the splat record's view depth (the value `depth` blends), 1/z_i the
 *                                         correctly rounded reciprocal; no background term.
 * With C > 128 (several channel chunks) chunk 0 writes them, as it writes colour and depth.
 *   f3dgs_forward_alpha_invdepth: f3dgs_forward_antialiased's arguments, then antialiasing (0: the default forward's
 *     opacities, else the antialiased forward's op_eff), out_alpha and out_invdepth (both required).  Colour, the
 *     feature map, depth, radii, the return value and the three buffers are bitwise those of f3dgs_forward / _f16 /
 *     _antialiased for the same arguments.
 *   f3dgs_backward_alpha_invdepth / f3dgs_backward_accum_alpha_invdepth: the arguments of f3dgs_backward_antialiased /
 *     f3dgs_backward_accum_antialiased (semantic_feature optional: given, the feature term of dL/dalpha is added;
 *     dL_dcamera optional), then antialiasing (0: the composite's opacity gradient goes straight to dL_dopacity, as in
 *     the default entries; else as in the _antialiased entries), dL_dalpha = dL/dA and dL_dinvdepth = dL/dI ([H,W]
 *     float32, both required).  With gA_p = dL_dalpha[p], gI_p = dL_dinvdepth[p] the composite adds
 *         dL/dalpha_i += gA_p T_final,p / (1 - alpha_i)        (the background term with bg.dL/dpix - gA_p),
 *         dL/dalpha_i += T_i (1/z_i - B_i) gI_p,   B_i = alpha_{i+1} / z_{i+1} + (1 - alpha_{i+1}) B_{i+1},   B_last = 0,
 *         dL/dz_i     -= sum_p w_ip gI_p / z_i^2,
 *     which reach dL_dopacity, dL_dmean2D, dL_dconic, dL_dz and through the preprocess dL_dmean3D, dL_dscale, dL_drot,
 *     dL_dcov3D, dL_dcamera and the densification statistics.  dL_dcolor and dL_dsemantic_feature are unchanged.  With
 *     dL_dalpha = dL_dinvdepth = 0 every output is bitwise that of the counterpart: f3dgs_backward[_f16], _cam[_f16],
 *     _feature_geometry or _antialiased (and their _accum twins) for the same remaining arguments.
 *   F3DGS_ERR_INVALID_ARGUMENT, before any launch, for a NULL plane, a plane overlapping another output (the forward's
 *     planes: out_color, out_feature_map, out_depth, radii or each other; the backward's plane gradients: any output),
 *     an unknown dtype code and whatever the counterpart rejects.
 * Buffers: the backward reads only what every forward stores (splat records, final_T, n_contrib); the planes are not
 * kept.  So the buffers of f3dgs_forward_alpha_invdepth and those of the counterpart forward with the same antialiasing
 * go to either backward, with bitwise equal gradients.  The antialiasing flag must match the forward's, as between the
 * _antialiased entries and the others. */
int f3dgs_forward_alpha_invdepth(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx,
                                 f3dgs_alloc_fn binning_alloc, void* binning_ctx,
                                 f3dgs_alloc_fn image_alloc, void* image_ctx,
                                 int P, int D, int M, int C,
                                 const float* background, int width, int height,
                                 const float* means3D, const float* shs, const float* colors_precomp,
                                 const void* semantic_feature, int semantic_feature_dtype, const float* opacities,
                                 const float* scales, float scale_modifier, const float* rotations,
                                 const float* cov3D_precomp,
                                 const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                 float tan_fovx, float tan_fovy, int prefiltered,
                                 float* out_color, void* out_feature_map, float* out_depth, int* radii,
                                 int debug, void* cuda_stream,
                                 int antialiasing, float* out_alpha, float* out_invdepth);
int f3dgs_backward_alpha_invdepth(int P, int D, int M, int R, int C,
                                  const float* background, int width, int height,
                                  const float* means3D, const float* shs, const float* colors_precomp,
                                  const void* semantic_feature, int semantic_feature_dtype,
                                  const float* scales, float scale_modifier, const float* rotations,
                                  const float* cov3D_precomp,
                                  const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                  float tan_fovx, float tan_fovy, const int* radii,
                                  char* geom_buffer, char* binning_buffer, char* image_buffer,
                                  const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                                  float dL_dfeaturepix_scale, const float* dL_depths,
                                  float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                                  float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                                  float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz,
                                  int debug, void* cuda_stream, float* dL_dcamera,
                                  int antialiasing, const float* dL_dalpha, const float* dL_dinvdepth);
int f3dgs_backward_accum_alpha_invdepth(int P, int D, int M, int R, int C,
                                        const float* background, int width, int height,
                                        const float* means3D, const float* shs, const float* colors_precomp,
                                        const void* semantic_feature, int semantic_feature_dtype,
                                        const float* scales, float scale_modifier, const float* rotations,
                                        const float* cov3D_precomp,
                                        const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                        float tan_fovx, float tan_fovy, const int* radii,
                                        char* geom_buffer, char* binning_buffer, char* image_buffer,
                                        const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                                        float dL_dfeaturepix_scale, const float* dL_depths, char* scratch,
                                        float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature,
                                        float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale,
                                        float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                                        void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera,
                                        int antialiasing, const float* dL_dalpha, const float* dL_dinvdepth);

/* ---- absolute-gradient densification statistic (opt-in; AbsGS, Ye et al., ACM MM 2024; gsplat's absgrad=True) ----
 * dL/dmean2D_i is a sum over the pixels p a view blends Gaussian i into of per-pixel terms t_ip = (t_x, t_y), in
 * dL_dmean2D's units (the 0.5 W, 0.5 H of the reference).  Terms of opposite sign cancel there, so a large Gaussian over
 * fine texture keeps a small ||dL/dmean2D|| and is never split ("gradient collision").  The _absgrad entries also give
 *     dL_dmean2D_abs[i] = ( sum_p |t_x|, sum_p |t_y|, 0 )                                   [P,3] float32
 *     grad_accum_abs[i] += sqrt(ax^2 + ay^2)   for radii_i > 0, (ax, ay) the first two columns   (accumulating entry)
 * from the backward composite's own reduction (each parked row of 32 per-pixel terms is summed twice, once as it is and
 * once as absolute values).  With the plane gradients t_ip includes their terms.  With the feature term of dL/dalpha
 * (semantic_feature given, C > 0) the colour walk and the feature walk each reduce their own terms, so the statistic is
 * sum_p |colour-walk term| + sum_p |feature-walk term|, which is AbsGS's value wherever one of the two is zero.
 *   f3dgs_backward_absgrad / f3dgs_backward_accum_absgrad: the arguments of f3dgs_backward_alpha_invdepth /
 *     f3dgs_backward_accum_alpha_invdepth, except that dL_dalpha and dL_dinvdepth may both be NULL (no planes; one
 *     alone is invalid), then dL_dmean2D_abs ([P,3], required).  The assigning entry adds into dL_dmean2D_abs as it
 *     adds into dL_dmean2D (the caller zeroes it; the third column stays 0).  The accumulating entry zeroes it itself
 *     and leaves this view's values in it, and takes grad_accum_abs ([P], optional; it needs grad_accum and denom),
 *     added to as grad_accum is.  Every other output is bitwise that of the counterpart entry: _alpha_invdepth with
 *     planes, otherwise f3dgs_backward[_f16], _cam[_f16], _feature_geometry or _antialiased (and their _accum twins).
 *   F3DGS_ERR_INVALID_ARGUMENT, before any launch, for a NULL dL_dmean2D_abs, a dL_dmean2D_abs or grad_accum_abs
 *     overlapping another output, grad_accum_abs without grad_accum / denom, one plane alone, and whatever the
 *     counterpart rejects. */
int f3dgs_backward_absgrad(int P, int D, int M, int R, int C,
                           const float* background, int width, int height,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const void* semantic_feature, int semantic_feature_dtype,
                           const float* scales, float scale_modifier, const float* rotations,
                           const float* cov3D_precomp,
                           const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                           float tan_fovx, float tan_fovy, const int* radii,
                           char* geom_buffer, char* binning_buffer, char* image_buffer,
                           const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                           float dL_dfeaturepix_scale, const float* dL_depths,
                           float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                           float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                           float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz,
                           int debug, void* cuda_stream, float* dL_dcamera,
                           int antialiasing, const float* dL_dalpha, const float* dL_dinvdepth,
                           float* dL_dmean2D_abs);
int f3dgs_backward_accum_absgrad(int P, int D, int M, int R, int C,
                                 const float* background, int width, int height,
                                 const float* means3D, const float* shs, const float* colors_precomp,
                                 const void* semantic_feature, int semantic_feature_dtype,
                                 const float* scales, float scale_modifier, const float* rotations,
                                 const float* cov3D_precomp,
                                 const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                 float tan_fovx, float tan_fovy, const int* radii,
                                 char* geom_buffer, char* binning_buffer, char* image_buffer,
                                 const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                                 float dL_dfeaturepix_scale, const float* dL_depths, char* scratch,
                                 float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature,
                                 float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale,
                                 float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                                 void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera,
                                 int antialiasing, const float* dL_dalpha, const float* dL_dinvdepth,
                                 float* dL_dmean2D_abs, float* grad_accum_abs);

/* ---- depth distortion loss (opt-in; Mip-NeRF 360's distortion term as 2DGS and gsplat's `distloss` use it on splats,
 * here in its L1 form on view depth) ----
 * For pixel p take the pairs i = 1..n the composite blends, in blend order, with w_i = alpha_i T_i and z_i the splat
 * record's view depth (the value `depth` blends).  Each tile list is sorted by z (the sort key's low word is the float
 * bits of z > 0), so z_i is non-decreasing along i and
 *     L_p = sum_i sum_j w_i w_j |z_i - z_j| = 2 sum_i w_i (z_i A_i - D_i),   A_i = sum_{j<i} w_j = 1 - T_i,
 *                                                                          D_i = sum_{j<i} w_j z_j.
 * It pulls each pixel's blend weights together along the ray, which removes semi-transparent floaters.  Ties in z add 0.
 * The loss weight, and any normalisation by scene scale, is the caller's.  With C > 128 chunk 0 writes the plane.
 *   f3dgs_forward_distortion: f3dgs_forward_antialiased's arguments, then antialiasing (as in
 *     f3dgs_forward_alpha_invdepth) and out_distortion ([H,W] float32, required).  Per blended pair the composite adds
 *     w (z (1 - T) - D) before D takes the pair, and writes twice the sum.  Colour, the feature map, depth, radii, the
 *     return value and the three buffers are bitwise those of the counterpart forward for the same arguments.
 *   f3dgs_backward_distortion / f3dgs_backward_accum_distortion: the arguments of f3dgs_backward_antialiased /
 *     f3dgs_backward_accum_antialiased (semantic_feature optional: given, the feature term of dL/dalpha is added;
 *     dL_dcamera optional), then antialiasing (as in the _alpha_invdepth entries), depth (the forward's depth plane
 *     [H,W], required), dL_ddistortion = dL/dL_p ([H,W] float32, required), dL_dmean2D_abs ([P,3], optional: NULL means
 *     no AbsGS statistic; otherwise as in the _absgrad entries) and, for the accumulating entry, grad_accum_abs ([P],
 *     optional, as in f3dgs_backward_accum_absgrad; it needs dL_dmean2D_abs).  With g = dL_ddistortion[p],
 *     Abar_i = sum_{j>i} w_j = T_{i+1} - T_final and Dbar_i = sum_{j>i} w_j z_j, the composite adds
 *         c_i = dL_p/dw_i = 2 [z_i (A_i - Abar_i) + Dbar_i - D_i],   D_i = depth[p] - Dbar_i - w_i z_i,
 *         dL/dalpha_i += T_i (c_i - B_i) g,   B_i = alpha_{i+1} c_{i+1} + (1 - alpha_{i+1}) B_{i+1},   B_last = 0,
 *         dL/dz_i     += 2 w_i (A_i - Abar_i) g.
 *     At ties in z this is the subgradient that orders the tied pairs by blend order (the later one counts as the
 *     farther).  The terms reach dL_dopacity, dL_dmean2D, dL_dconic, dL_dz and through the preprocess dL_dmean3D,
 *     dL_dscale, dL_drot, dL_dcov3D, dL_dcamera and the densification statistics; under AbsGS each pixel's 2-D mean term
 *     includes the distortion's share.  dL_dcolor and dL_dsemantic_feature are unchanged.  With dL_ddistortion = 0
 *     every output is bitwise that of the counterpart: f3dgs_backward[_f16], _cam[_f16], _feature_geometry or
 *     _antialiased (and their _accum twins), or the _absgrad entries without planes when dL_dmean2D_abs is given.
 *     Distortion and the _alpha_invdepth planes do not combine in one call.
 *   F3DGS_ERR_INVALID_ARGUMENT, before any launch, for a NULL out_distortion, depth or dL_ddistortion, an out_distortion
 *     overlapping another output, a depth or dL_ddistortion overlapping an output, grad_accum_abs without
 *     dL_dmean2D_abs, and whatever the counterpart rejects.
 * Buffers: the backward reads only what every forward stores, plus `depth`.  So the buffers of any forward with the
 * same antialiasing go to it, with that forward's depth plane. */
int f3dgs_forward_distortion(f3dgs_alloc_fn geometry_alloc, void* geometry_ctx,
                             f3dgs_alloc_fn binning_alloc, void* binning_ctx,
                             f3dgs_alloc_fn image_alloc, void* image_ctx,
                             int P, int D, int M, int C,
                             const float* background, int width, int height,
                             const float* means3D, const float* shs, const float* colors_precomp,
                             const void* semantic_feature, int semantic_feature_dtype, const float* opacities,
                             const float* scales, float scale_modifier, const float* rotations,
                             const float* cov3D_precomp,
                             const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                             float tan_fovx, float tan_fovy, int prefiltered,
                             float* out_color, void* out_feature_map, float* out_depth, int* radii,
                             int debug, void* cuda_stream,
                             int antialiasing, float* out_distortion);
int f3dgs_backward_distortion(int P, int D, int M, int R, int C,
                              const float* background, int width, int height,
                              const float* means3D, const float* shs, const float* colors_precomp,
                              const void* semantic_feature, int semantic_feature_dtype,
                              const float* scales, float scale_modifier, const float* rotations,
                              const float* cov3D_precomp,
                              const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                              float tan_fovx, float tan_fovy, const int* radii,
                              char* geom_buffer, char* binning_buffer, char* image_buffer,
                              const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                              float dL_dfeaturepix_scale, const float* dL_depths,
                              float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                              float* dL_dsemantic_feature, float* dL_dmean3D, float* dL_dcov3D,
                              float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dz,
                              int debug, void* cuda_stream, float* dL_dcamera,
                              int antialiasing, const float* depth, const float* dL_ddistortion,
                              float* dL_dmean2D_abs);
int f3dgs_backward_accum_distortion(int P, int D, int M, int R, int C,
                                    const float* background, int width, int height,
                                    const float* means3D, const float* shs, const float* colors_precomp,
                                    const void* semantic_feature, int semantic_feature_dtype,
                                    const float* scales, float scale_modifier, const float* rotations,
                                    const float* cov3D_precomp,
                                    const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                    float tan_fovx, float tan_fovy, const int* radii,
                                    char* geom_buffer, char* binning_buffer, char* image_buffer,
                                    const float* dL_dpix, const void* dL_dfeaturepix, int dL_dfeaturepix_dtype,
                                    float dL_dfeaturepix_scale, const float* dL_depths, char* scratch,
                                    float* dL_dopacity, float* dL_dcolors_precomp, float* dL_dsemantic_feature,
                                    float* dL_dmean3D, float* dL_dcov3D_precomp, float* dL_dsh, float* dL_dscale,
                                    float* dL_drot, float* dL_dmean2D_out, float* grad_accum, float* denom,
                                    void* composite_done_event, int debug, void* cuda_stream, float* dL_dcamera,
                                    int antialiasing, const float* depth, const float* dL_ddistortion,
                                    float* dL_dmean2D_abs, float* grad_accum_abs);

/* ---- feature lifting (no reference counterpart): training-free back-projection of 2-D feature maps onto Gaussians ----
 * The buffers and R are those of an f3dgs_forward / _f16 / _antialiased / _alpha_invdepth of this view at width x height
 * (any C of that forward, 0 included); feature_map [C,H,W] is a map at that resolution, 1 <= C <= F3DGS_MAX_FEATURE_DIM.
 * ACCUMULATES:  feature_sum[P,C] += sum_p w_ip * feature_map[:,p];   weight_sum[P] += sum_p w_ip,
 * w_ip = the blend weight alpha*T of Gaussian i at pixel p (the backward's unwound T: equal to the forward's blend weight
 * to a few ulp).  Over views, feature_sum / weight_sum is the blend-weighted mean of the maps per Gaussian.  The result
 * equals f3dgs_backward's dL_dsemantic_feature and dL_dcolor[:,0] for dL_dfeaturepix = feature_map, dL_dpix = the planes
 * (1, 0, 0) and dL_depths = 0, up to the order of the float reductions, without the geometric gradients.
 * The outputs must not overlap the map or each other.  P == 0 or R == 0 launches nothing.  The instance lists (136
 * bytes per (instance, 8x4 block) of capacity) are stream-ordered scratch of the device's default memory pool.
 *   f3dgs_lift_features_accum_f16: feature_map holds IEEE binary16 bits (a saved *_fmap_CxHxW.pt as loaded), upcast
 *   exactly; the result is that of the float32 call on the upcast map.  Validates as the float32 call, with the map's
 *   2-byte size in the overlap checks. */
int f3dgs_lift_features_accum(int P, int R, int C, int width, int height, char* geom_buffer, char* binning_buffer,
                              char* image_buffer, const float* feature_map, float* feature_sum, float* weight_sum,
                              void* cuda_stream);
int f3dgs_lift_features_accum_f16(int P, int R, int C, int width, int height, char* geom_buffer, char* binning_buffer,
                                  char* image_buffer, const uint16_t* feature_map, float* feature_sum,
                                  float* weight_sum, void* cuda_stream);

/* ---- per-Gaussian blend-weight scores (no reference counterpart): the statistics compaction methods prune by -------
 * The buffers and R are those of an f3dgs_forward / _f16 / _antialiased / _alpha_invdepth of this view at width x height
 * (any C of that forward, 0 included; an antialiased forward scores the antialiased model).  ACCUMULATES:
 *   weight_sum[P]  += sum_p w_ip                          (LightGaussian's global significance without its volume
 *                                                          factor, Mini-Splatting's importance)
 *   max_weight[P]   = max(max_weight, max_p w_ip)         (RadSplat's score)
 *   pixel_count[P] += #{p : Gaussian i blended into p}    (LightGaussian's hit count), exact
 * w_ip = the blend weight alpha*T of Gaussian i at pixel p (the backward's unwound T, the value
 * f3dgs_lift_features_accum's weight_sum adds: equal to the forward's blend weight to a few ulp); the pairs counted are
 * exactly those the forward composited.  max_weight must hold values >= 0 (zeros to start): it is updated with an
 * integer max on the float bits, so it is exact and does not depend on the order of the views.  weight_sum equals
 * f3dgs_lift_features_accum's on the same buffers up to the order of the float reductions.  The three outputs must not
 * overlap.  P == 0 or R == 0 launches nothing.  The call allocates nothing: one kernel, the geometry walk of the
 * backward without its instance lists or feature kernel, and no upstream gradient is read. */
int f3dgs_gaussian_scores_accum(int P, int R, int width, int height, char* geom_buffer, char* binning_buffer,
                                char* image_buffer, float* weight_sum, float* max_weight, int64_t* pixel_count,
                                void* cuda_stream);

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
/* Training float16 feature fields.
 *   f3dgs_feature_resize_fwd_f16        feature_map [C,H,W] float16; gt float32 or NULL.
 *   f3dgs_feature_resize_fwd_f16_f16gt  feature_map and gt float16 (gt required).
 *       The result (out and loss_sum, float32) is that of f3dgs_feature_resize_fwd applied to the exactly upcast inputs.
 *   f3dgs_feature_resize_bwd_f16        dL_dfeature_map [C,H,W] float16 = half_rn(out_scale * f3dgs_feature_resize_bwd
 *       (dout)) elementwise (+-inf beyond 65504, as torch's .half()); out_scale finite and nonzero.  An L1 loss passes
 *       grad_scale = 1 to the forward (exact signs), out_scale = 1, and hands the map to f3dgs_backward_f16 with the
 *       scale weight / (C*Hg*Wg), which float16 alone cannot hold.
 * They validate as their float32 twins, and also reject an output that overlaps an input (2-byte sizes for float16). */
int f3dgs_feature_resize_fwd_f16(int C, int H, int W, int Hg, int Wg, const uint16_t* feature_map, const float* gt,
                                 float grad_scale, float* out, float* loss_sum, void* cuda_stream);
int f3dgs_feature_resize_fwd_f16_f16gt(int C, int H, int W, int Hg, int Wg, const uint16_t* feature_map,
                                       const uint16_t* gt, float grad_scale, float* out, float* loss_sum,
                                       void* cuda_stream);
int f3dgs_feature_resize_bwd_f16(int C, int H, int W, int Hg, int Wg, const float* dout, float out_scale,
                                 uint16_t* dL_dfeature_map, void* cuda_stream);

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

/* ---- text query: LSeg's segmentation head on a rendered or saved feature map; render_edit's CLIP-text selection of
 * Gaussians (gaussian_renderer/__init__.py:58-170) -----------------------------------------------------------------
 * x [C,N] (a map [C,H,W] as N = H*W columns, or per-Gaussian features transposed to [C,P]), weight [D,C] (the
 * CNN_decoder conv weight as contiguous memory) or NULL (no decoder, D == C), bias [D] or NULL (only with weight),
 * text [K,D] embeddings, positive [K] (nonzero = positive prompt) or NULL.  1 <= K <= 256, 1 <= D <= 4096, N >= 0
 * (N == 0 launches nothing), 1 <= C <= 256 with a decoder.  For every column n:
 *     y = weight x_n + bias (x_n without weight);  l_k = logit_scale * <y / max(||y||, 1e-12), t_k / max(||t_k||, 1e-12)>
 *   f3dgs_feature_query  labels[N] int64 = argmax_k l_k (first maximal index, as torch.argmax; an all-NaN column
 *                        gives 0); prob[N] = sum over positive k of softmax_k(l) (fp32, max-subtracted; exactly 1 when
 *                        every prompt is positive; needs positive); logits[K,N] = l.  Each output may be NULL, but
 *                        one is required; every element of a requested one is written; none may overlap an input or
 *                        another output; logit_scale must be finite.
 *   f3dgs_feature_query_f16x  x [C,N] float16 (a saved map): the result of f3dgs_feature_query for the exactly upcast
 *                        x, bitwise.  Validates as f3dgs_feature_query, with x's 2-byte size in the overlap checks.
 * Both products use TF32 operands (rounded to nearest) with fp32 accumulation, ||y||^2 is summed in fp32 before any
 * rounding; nothing of size D*N is stored, and results are bitwise reproducible whichever outputs are requested. */
int f3dgs_feature_query(int C, int D, int K, int N, const float* weight, const float* bias, const float* x,
                        const float* text, float logit_scale, const uint8_t* positive, int64_t* labels, float* prob,
                        float* logits, void* cuda_stream);
int f3dgs_feature_query_f16x(int C, int D, int K, int N, const float* weight, const float* bias, const uint16_t* x,
                             const float* text, float logit_scale, const uint8_t* positive, int64_t* labels,
                             float* prob, float* logits, void* cuda_stream);

/* ---- PCA picture of a feature map: render.py's feature_visualize_saving (render.py:147-180) -----------------------
 * x [C,N] (a map [C,H,W] as N = H*W pixels, p = y*W + x), 3 <= C <= 1024, N >= 7 (n = ceil(N/3) >= 3 samples: the
 * pixels p = 3s).  With xh_p = x_p / max(||x_p||, 1e-12):
 *   f3dgs_feature_pca_moments  mean[C] float32 = the mean of xh over the samples; cov[C,C] float64 =
 *                              sum over samples of (xh - mean)(xh - mean)^T / (n - 1), symmetric.  Centred on load,
 *                              fp32 FMA over blocks of 2048 samples, blocks and CTA partials added in fp64 in a fixed order.
 *   (caller)                   the unit eigenvectors c_1..c_3 of cov for its three largest eigenvalues, descending, each
 *                              signed so that its entry of largest |value| (the first such) is positive, as float32
 *                              components[3,C].  This library has no eigensolver: LAPACK dsyevd (or cuSOLVER syevd) on
 *                              cov is the intended one; cov is fp64 so that the solver sees the accumulated precision.
 *   f3dgs_feature_pca_range    range[2] float32 = np.percentile(t, [1, 99]) (linear) of the 3n values
 *                              t = c_k . (xh_s - mean), written on the device (no host sync).
 *   f3dgs_feature_pca_image    image[N,3] float32: clamp((c_k . (xh_p - mean) - lo) / (hi - lo), 0, 1) for every pixel
 *                              (lo, hi = range, read on the device; hi == lo gives the IEEE result, NaN stays NaN).
 * scratch is f3dgs_feature_pca_scratch_bytes(C, N) bytes of device memory, 256-byte aligned, for the moments and range
 * calls (the size does not depend on x's dtype; 0 for sizes out of range, and 0 with f3dgs_last_error() set if the size
 * query of the device sort fails).  No output may overlap an input, the scratch or another output.  The _f16x variants
 * take x as IEEE binary16 bits and give bitwise the result for the exactly upcast x; they validate as their float32
 * twins, with x's 2-byte size in the overlap checks.  Every call is stream-ordered, launches only device work and is
 * bitwise reproducible; a map is read once by the image call and about once per pass by the other two. */
size_t f3dgs_feature_pca_scratch_bytes(int C, int N);
int f3dgs_feature_pca_moments(int C, int N, const float* x, char* scratch, float* mean, double* cov, void* cuda_stream);
int f3dgs_feature_pca_moments_f16x(int C, int N, const uint16_t* x, char* scratch, float* mean, double* cov,
                                   void* cuda_stream);
int f3dgs_feature_pca_range(int C, int N, const float* x, const float* mean, const float* components, char* scratch,
                            float* range, void* cuda_stream);
int f3dgs_feature_pca_range_f16x(int C, int N, const uint16_t* x, const float* mean, const float* components,
                                 char* scratch, float* range, void* cuda_stream);
int f3dgs_feature_pca_image(int C, int N, const float* x, const float* mean, const float* components,
                            const float* range, float* image, void* cuda_stream);
int f3dgs_feature_pca_image_f16x(int C, int N, const uint16_t* x, const float* mean, const float* components,
                                 const float* range, float* image, void* cuda_stream);

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
/* f3dgs_adam_step of an IDENTITY group (kind must be F3DGS_PARAM_IDENTITY) that also keeps a float16 working copy: in the
 * same pass, param_f16[n] (IEEE binary16 bits) = the updated param rounded to nearest even (torch's .half()).  param,
 * exp_avg and exp_avg_sq are bitwise those of f3dgs_adam_step and stay float32 (the master weights); param_f16 must not
 * overlap the other buffers.  For float16 feature fields: the rasterizer reads the copy, the optimizer the master. */
int f3dgs_adam_step_f16out(int kind, size_t n, int M, float* param, const float* grad_activated, float* exp_avg,
                           float* exp_avg_sq, uint16_t* param_f16, float lr, float beta1, float beta2, float eps,
                           int step, void* cuda_stream);
/* Sparse Adam (the upstream 3DGS rasterizer's SparseGaussianAdam): f3dgs_adam_step / f3dgs_adam_step_f16out on the rows
 * of P Gaussians marked in visible[P] (bytes, nonzero = visible) only.  The raw parameter is P rows of n / P elements:
 * SIGMOID 1, EXP 3, NORMALIZE4 4, SH_DC 3, SH_REST 3 (M - 1), IDENTITY any width; so P >= 1 and n % P == 0.  A visible
 * row's param, exp_avg, exp_avg_sq (and param_f16) are bitwise those of the dense entry; every other row is neither read
 * nor written, whatever its gradient holds.  Bias correction:
 *   step >= 1  as the dense entries, with the group's step count (it advances on every step, visible or not: one step
 *              counter per parameter, as torch's SparseAdam);
 *   step == 0  none (lr / (1 - b1^t) = lr, sqrt(1 - b2^t) = 1): upstream SparseGaussianAdam's update
 *              m = b1 m + (1 - b1) g, v = b2 v + (1 - b2) g^2, p -= lr m / (sqrt(v) + eps).
 * n == 0 is a no-op (pointers and P are not checked then).  The _f16out twin takes IDENTITY only, and its param_f16 must
 * not overlap the other buffers. */
int f3dgs_adam_step_masked(int kind, size_t n, int P, int M, float* param, const float* grad_activated, float* exp_avg,
                           float* exp_avg_sq, const uint8_t* visible, float lr, float beta1, float beta2, float eps,
                           int step, void* cuda_stream);
int f3dgs_adam_step_masked_f16out(int kind, size_t n, int P, int M, float* param, const float* grad_activated,
                                  float* exp_avg, float* exp_avg_sq, const uint8_t* visible, uint16_t* param_f16,
                                  float lr, float beta1, float beta2, float eps, int step, void* cuda_stream);

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
 * AbsGS's split rule is the same pair with another plan:
 *   f3dgs_densify_plan_absgrad  f3dgs_densify_plan's arguments, then grad_accum_abs ([P], required; the statistic of
 *                        f3dgs_backward_accum_absgrad) and abs_grad.  With ga = grad_accum_abs / denom (0 where NaN):
 *                          split  ga >= abs_grad && smax > dense_scale
 *                        clone and prune are unchanged.  (gsplat's variant, the abs statistic for both decisions, is
 *                        f3dgs_densify_plan with grad_accum_abs in place of grad_accum.)
 *
 * Pruning from a caller's mask is the same pair with another plan:
 *   f3dgs_prune_plan     keeps row i iff keep[i] != 0 (keep: P bytes of device memory, any nonzero byte keeps) and
 *                        writes counts = {A, 0, 0, 0}, A the rows kept.  scratch is f3dgs_densify_scratch_bytes(P)
 *                        bytes; keep and counts must not overlap its flags.  f3dgs_densify_apply with the host copy
 *                        of counts and normals == NULL then writes the A kept rows of every field, in order, bitwise.
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
int f3dgs_densify_plan_absgrad(int P, const float* grad_accum, const float* denom, const float* raw_opacity,
                               const float* raw_scaling, float max_grad, float dense_scale, float min_opacity,
                               float max_world_scale, char* scratch, int32_t* counts, void* cuda_stream,
                               const float* grad_accum_abs, float abs_grad);
int f3dgs_densify_apply(int P, int M, int C, const char* scratch, const int32_t counts[4], const float* normals,
                        const f3dgs_gaussian_fields src[3], const f3dgs_gaussian_fields dst[3], void* cuda_stream);
int f3dgs_prune_plan(int P, const uint8_t* keep, char* scratch, int32_t* counts, void* cuda_stream);
int f3dgs_reset_opacity(int P, float* raw_opacity, float* exp_avg, float* exp_avg_sq, float ceiling, void* cuda_stream);

/* ---- fixed-budget densification: 3DGS-MCMC (Kheradmand et al., NeurIPS 2024; the official code's relocate_gs,
 * add_new_gs and position noise, gsplat's MCMCStrategy) ------------------------------------------------------------
 * Fields as for f3dgs_densify_apply: fields[0] the raw parameters, [1] exp_avg, [2] exp_avg_sq.  The caller draws every
 * index and normal (e.g. torch.multinomial over alive_opacity / its sum, torch.randn), so a run is reproducible from its
 * generator.  With o = sigmoid(raw_opacity) (bitwise torch.sigmoid) and s = expf(raw_scaling):
 *   relocation rule  a source drawn c >= 1 times in a call ends as N = min(c + 1, 51) identical Gaussians, each with
 *                      o' = 1 - (1 - o)^(1/N)                     (evaluated as -expm1(log1p(-o) / N))
 *                      s' = s * o / D(o', N),  D(x, N) = sum_{j=1..N} C(N,j) (-1)^(j-1) x^j / sqrt(j)
 *                    in double; o' is then clamped to [min_opacity, 1 - FLT_EPSILON] (s' keeps the unclamped o'), and
 *                    raw_opacity = logit(o'), raw_scaling = log(s') are rounded to float once.  1 - (1 - o')^N = o
 *                    before the clamp.
 *   f3dgs_mcmc_plan      dead = (o <= min_opacity).  Writes index[P] = the dead indices ascending, then the alive ones
 *                        ascending; alive_opacity[0 .. P - n_dead) = o of the alive ones in that order; *n_dead (device
 *                        int32).  index and alive_opacity are P elements each; n_dead is the only count to read back.
 *   f3dgs_mcmc_relocate  in place, P unchanged: for each of the n draws j, row dead[j] takes every raw field of row
 *                        src[j] with (o', s'), row src[j] takes (o', s'), and src[j]'s exp_avg and exp_avg_sq are zeroed
 *                        in all seven fields.  The dead rows' moments are left as they are, as the reference does: it
 *                        resets the optimizer state of the sources only.  semantic_feature_f16 (NULL, or [P,C] IEEE
 *                        binary16 bits): the dead rows get their new features rounded to nearest even (torch's .half()).
 *                        Contract: the dead[] are distinct and no src[j] is a dead row; src[] may repeat.
 *   f3dgs_mcmc_add       out of place: dst has P + n rows.  Row i < P is src row i, except that a drawn row gets
 *                        (o', s') and zero moments; row P + j is a copy of src row src[j] with (o', s') and zero moments.
 *                        Every src element is read at most once and every dst element written once.  No dst field may
 *                        overlap a src field, src[] or the scratch.
 *   An index outside [0, P) in dead[] or src[] makes relocate and add write nothing to the caller's buffers (checked on
 *   the device before the first write).  0 <= n <= P.  scratch: f3dgs_mcmc_scratch_bytes(P) bytes of device memory,
 *   256-byte aligned, shared by the three calls (not kept between them).
 *   f3dgs_mcmc_inject_noise  xyz[P,3] += R diag(s^2) R^T (eps * g * scale), g = 1 / (1 + exp(-100 ((1 - o) - 0.995))),
 *                        R the rotation of the normalised quaternion (w, x, y, z), eps [P,3] the caller's normals;
 *                        computed in double and rounded once.  The reference's scale is noise_lr * xyz_lr with
 *                        noise_lr = 5e5, applied after every optimizer step.
 * All calls are stream-ordered without host sync and bitwise deterministic.  3 P (3 (P + n) for add, 4 P for the
 * noise) must not exceed INT_MAX; scale and
 * min_opacity must be finite.  f3dgs_mcmc_scratch_bytes returns 0 for P <= 0, and 0 with f3dgs_last_error() set if the
 * size query fails. */
size_t f3dgs_mcmc_scratch_bytes(int P);
int f3dgs_mcmc_plan(int P, const float* raw_opacity, float min_opacity, char* scratch, int32_t* n_dead, int32_t* index,
                    float* alive_opacity, void* cuda_stream);
int f3dgs_mcmc_relocate(int P, int M, int C, int n, const int32_t* dead, const int32_t* src, float min_opacity,
                        const f3dgs_gaussian_fields fields[3], uint16_t* semantic_feature_f16, char* scratch,
                        void* cuda_stream);
int f3dgs_mcmc_add(int P, int M, int C, int n, const int32_t* src, float min_opacity,
                   const f3dgs_gaussian_fields src_fields[3], const f3dgs_gaussian_fields dst_fields[3], char* scratch,
                   void* cuda_stream);
int f3dgs_mcmc_inject_noise(int P, float* xyz, const float* raw_opacity, const float* raw_scaling,
                            const float* raw_rotation, const float* eps, float scale, void* cuda_stream);

/* ---- 3D smoothing filter: Mip-Splatting (Yu et al., CVPR 2024; the official scene/gaussian_model.py
 * compute_3D_filter, get_opacity_with_3D_filter, get_scaling_with_3D_filter, reset_opacity) ------------------------
 * Each Gaussian gets a world-space filter size f from the highest sampling rate any training camera has at it; the
 * rasterizer is then called with the filtered opacity and scales, so that no Gaussian is smaller than the training
 * views could sample (no needles when rendering closer or at a higher resolution than any training view).
 *   f3dgs_filter3d_compute  viewmatrices [V,16] (the rasterizer's viewmatrix, W2C^T), intrinsics [V,4] = (fx, fy, W, H)
 *                        with fx = W / (2 tanfovx), fy = H / (2 tanfovy) as floats.  For Gaussian i with mean x and
 *                        camera v: c = x @ vm[:3,:3] + vm[3,:3] (fixed fma order), zc = max(c.z, 0.001),
 *                        px = c.x / zc * fx + W / 2, py = c.y / zc * fy + H / 2; v sees i when c.z > 0.2 and
 *                        -0.15 W <= px <= 1.15 W and -0.15 H <= py <= 1.15 H (margins rounded from double once).
 *                        d_i = min(100000, min over the cameras that see i of zc); a Gaussian no camera sees takes the
 *                        max d of the seen ones.  filter[i] = d_i * (1 / focal) * sqrt(0.2) in float, focal = max fx
 *                        (fx only, as the official code).  *n_seen (device int32) = the number of seen Gaussians; when
 *                        it is 0 the filter is meaningless (the official code fails there).  Bitwise deterministic and
 *                        independent of the camera order.  scratch: f3dgs_filter3d_scratch_bytes(P) bytes of device
 *                        memory (returns 0 for P <= 0); filter, n_seen and scratch must not overlap each other or an
 *                        input.  V >= 1.
 *   f3dgs_filter3d_apply  o, s the activated opacity [P] and scales [P,3]: opacity_out = o * coef and
 *                        scales_out = sqrt(s^2 + f^2) per axis, with det1 = s0^2 s1^2 s2^2, det2 = prod (s_k^2 + f^2)
 *                        and coef = sqrt(det1 / det2): bitwise the official float32 torch formula (torch's .prod(dim=1)
 *                        order, no contraction).  The outputs must not overlap each other or an input.
 *   f3dgs_filter3d_apply_backward  the gradients w.r.t. (o, s) from those w.r.t. (opacity_out, scales_out):
 *                        dL_dopacity = dL_dopacity_f * coef,
 *                        dL_dscales_k = dL_dscales_f_k * s_k / s_f_k + dL_dopacity_f * o_f * f^2 / (s_k s_f_k^2),
 *                        the second term 0 where o_f == 0 (an underflowed det1 or s_k == 0 gives no NaN).  The filter
 *                        gets no gradient.  dL_dopacity may be dL_dopacity_f and dL_dscales may be dL_dscales_f (in
 *                        place); no other overlap is allowed.
 *   f3dgs_reset_opacity_filter3d  f3dgs_reset_opacity of the filtered opacity, in place: with o = sigmoid(raw_opacity),
 *                        s = expf(raw_scaling) and coef as above, raw_opacity <- logit(min(o * coef, ceiling) / coef)
 *                        (NaN propagates); exp_avg and exp_avg_sq of the opacity [P] are zeroed.  Where coef == 0 the
 *                        official formula is 0 / 0; there the unfiltered reset's logit(min(o, ceiling)) is written.
 *                        raw_opacity, exp_avg and exp_avg_sq must not overlap each other, raw_scaling or filter.
 * All calls are stream-ordered without host sync.  0 <= 3 P <= INT_MAX; P == 0 is a no-op. */
size_t f3dgs_filter3d_scratch_bytes(int P);
int f3dgs_filter3d_compute(int P, int V, const float* means3D, const float* viewmatrices, const float* intrinsics,
                           float* filter, int32_t* n_seen, char* scratch, void* cuda_stream);
int f3dgs_filter3d_apply(int P, const float* opacity, const float* scales, const float* filter, float* opacity_out,
                         float* scales_out, void* cuda_stream);
int f3dgs_filter3d_apply_backward(int P, const float* opacity, const float* scales, const float* filter,
                                  const float* dL_dopacity_f, const float* dL_dscales_f, float* dL_dopacity,
                                  float* dL_dscales, void* cuda_stream);
int f3dgs_reset_opacity_filter3d(int P, float* raw_opacity, const float* raw_scaling, const float* filter,
                                 float* exp_avg, float* exp_avg_sq, float ceiling, void* cuda_stream);

/* ---- vector quantisation: k-means codebooks of per-row features (LightGaussian, NeurIPS 2024; CompGS, ECCV 2024) ----
 * Rows x [P,D] float32, a codebook c [K,D] float32 and codes code [P] int32, all row-major.  1 <= D <= 4096,
 * 1 <= K <= 65536, P >= 0; P == 0 launches nothing.
 *   f3dgs_vq_assign      code[i] = argmin_k (||c_k||^2 - 2 x_i . c_k).  The products run on the tensor cores in TF32:
 *                        x and c rounded to nearest (cvt.rna), fp32 accumulation, as f3dgs_feature_query; ||c_k||^2 is
 *                        summed in fp32 from the unrounded codebook.  Ties go to the lower index.  A NaN score loses to
 *                        every number, so a row whose scores are all NaN (a NaN in x) gets code 0.  Only the codes reach
 *                        memory.  Error bound: with d(x, c) = ||x - c||^2 in exact arithmetic on the float32 inputs,
 *                        cmax = max_k ||c_k||, u = 2^-11 (TF32 rounding) and g = (D + 8) 2^-22 (the fp32 sums of D
 *                        terms as the tensor cores form them, products exact and each k8 block added with alignment
 *                        and truncation; the norm sum; the final subtraction), every row satisfies
 *                          d(x, c_code) - min_k d(x, c_k) <= (4 (2u + u^2) + 4 g (1 + u)^2) ||x|| cmax + 2 g cmax^2
 *                        i.e. (2^-8 + 2^-20 + 4 g (1 + 2^-11)^2) ||x|| cmax + 2 g cmax^2: twice (for the chosen code and
 *                        the best one) the rounding of two products x . c (Cauchy-Schwarz) plus the fp32 sums.  code
 *                        must not overlap x or the codebook.  The rounded codebook (K D floats, padded) comes from the
 *                        device's default memory pool.
 *   f3dgs_vq_plan        a stable sort of the row indices by code and the segment offsets of each code, written to
 *                        scratch (f3dgs_vq_scratch_bytes(P, K) bytes of device memory, 256-byte aligned).  The plan stays
 *                        valid while the codes do not change: update and codebook_grad only read it.  A code outside
 *                        [0, K) is detected on the device: every update or codebook_grad over that plan then writes
 *                        nothing.  scratch must not overlap code.
 *   f3dgs_vq_update      in place: c_k = sum w_i x_i / sum w_i over the plan's rows of code k, the sums in double,
 *                        rounded once; weights [P] (NULL: all ones) must be finite and >= 0: otherwise (checked on the
 *                        device before any write) the call writes nothing.  A code with zero total weight keeps its row
 *                        bitwise.
 *   f3dgs_vq_codebook_grad  dL_dcodebook[k] = sum dL_dx_i over the plan's rows of code k, in double, rounded once,
 *                        written (0 for an empty code): the chain rule of decode's gather.
 *   Both reductions use no float atomics and a fixed order (set by P and the codes), and spread every code's rows over
 *   CTAs of at most 512 rows, one code holding every row included.  Their partial sums (8 D (P / 256 + 1) bytes) come
 *   from the device's default memory pool.  codebook (update) and dL_dcodebook must not overlap an input or the scratch.
 *   f3dgs_vq_decode      out[i, :] = c[code[i], :], float32; f3dgs_vq_decode_f16out writes the IEEE binary16 bits of
 *                        half_rn(c[code[i], :]), bitwise torch's c.half()[code].  A code outside [0, K) decodes to a NaN
 *                        row.  out must not overlap the codebook or code.
 * F3DGS_ERR_INVALID_ARGUMENT, before any CUDA call, for sizes out of range, a NULL pointer (with P > 0) or an overlap.
 * Stream-ordered without host sync; every result is bitwise reproducible.  f3dgs_vq_scratch_bytes returns 0 for P <= 0
 * or K out of range, and 0 with f3dgs_last_error() set if the size query fails. */
size_t f3dgs_vq_scratch_bytes(int P, int K);
int f3dgs_vq_assign(int P, int K, int D, const float* x, const float* codebook, int32_t* code, void* cuda_stream);
int f3dgs_vq_plan(int P, int K, const int32_t* code, char* scratch, void* cuda_stream);
int f3dgs_vq_update(int P, int K, int D, const float* x, const float* weights, const char* scratch, float* codebook,
                    void* cuda_stream);
int f3dgs_vq_codebook_grad(int P, int K, int D, const float* dL_dx, const char* scratch, float* dL_dcodebook,
                           void* cuda_stream);
int f3dgs_vq_decode(int P, int K, int D, const float* codebook, const int32_t* code, float* out, void* cuda_stream);
int f3dgs_vq_decode_f16out(int P, int K, int D, const float* codebook, const int32_t* code, uint16_t* out,
                           void* cuda_stream);

/* ---- neighbour graphs of Gaussians: exact k-NN, its reverse lists, total variation of a feature field over it, and
 * the neighbour fill of low-weight rows ---------------------------------------------------------------------------
 * P points [P,3] float32, 1 <= k <= 32, P k <= 2^31 - 1; P == 0 launches nothing.  Graph arrays are row-major [P,k].
 *   f3dgs_knn_graph      idx [P,k] int32 and dist2 [P,k] float32 in input row order: row i holds the k nearest points
 *                        j != i (exclusion by index, so a coincident point is a neighbour at distance 0), ascending by the
 *                        pair (dist2, j) compared lexicographically, so ties go to the lower index.  dist2 is
 *                        f3dgs_knn_mean_dist's one expression, fma(dz, dz, fma(dy, dy, dx * dx)) of the rounded
 *                        differences candidate - query per axis.  Entries past P - 1 are idx = -1, dist2 = +inf.  order
 *                        [P] int32 receives the Morton order of the search (a permutation of [0, P)), in which rows
 *                        close in space are close in memory.  The result is EXACT: the search prunes a box only when its
 *                        distance, a lower bound on the rounded distance of every point inside (rounding is monotone),
 *                        is above the current k-th distance.  No float atomics: bitwise reproducible, and a permutation
 *                        of the points permutes the rows (dist2 is unchanged).  Results are specified for finite
 *                        coordinates only.  idx, dist2 and order must not overlap each other, points or scratch.
 *   f3dgs_knn_reverse    the transpose of idx in CSR form: sources[offsets[n] .. offsets[n+1]) are the rows i with n in
 *                        idx[i], ascending (a stable radix sort of the (neighbour, source) pairs).  Entries of idx outside
 *                        [0, P), -1 among them, are dropped; offsets[P] is the number of valid entries and sources past it
 *                        are -1.  offsets [P+1] and sources [P k] int32 must not overlap each other, idx or scratch.
 *   Both take scratch of f3dgs_knn_graph_scratch_bytes(P, k) bytes of device memory, 256-byte aligned (0 for sizes out
 *   of range, and 0 with f3dgs_last_error() set if a size query of the device sort fails).
 *   f3dgs_feature_tv_accum  total variation of features f [P,C] float32 (1 <= C <= F3DGS_MAX_FEATURE_DIM) over the graph's
 *                        valid edges E (n_edges = |E|, given by the caller):
 *                          L = weight / (|E| C) * sum_{(i,j) in E} sum_c |f_ic - f_jc|
 *                          grad_i += float(n_i) * s,   s = (float)(weight / (|E| C)),
 *                          n_i = sum_{j in N(i)} sign(f_i - f_j) - sum_{i' in R(i)} sign(f_i' - f_i),  sign(0) = 0
 *                        with N from idx and R from the reverse lists (offsets, sources).  n_i is an integer counted
 *                        exactly; the product and the add are each rounded to nearest (no fma), so grad is defined
 *                        bitwise and is ADDED to.  *loss (device double) = L, from per-row float64 sums reduced in a fixed
 *                        order.  order [P] (may be NULL: row order) is the walk order over rows; the results do not
 *                        depend on it.  n_edges == 0: *loss = 0 and grad is untouched.  P + 1024 doubles of partial sums
 *                        come from the device's default memory pool (F3DGS_ERR_ALLOC if that fails).  grad and loss must
 *                        not overlap each other or an input; weight must be finite.
 *   f3dgs_feature_fill   out [P,C] = features, except that a row i with weights[i] <= min_weight and at least one
 *                        neighbour j with weights[j] > min_weight becomes sum_j w_j f_j / sum_j w_j over those
 *                        neighbours, both sums in double in neighbour order, the quotient rounded once to float32.
 *                        weights [P] float32; min_weight must not be NaN; out must not overlap features, weights or idx.
 * F3DGS_ERR_INVALID_ARGUMENT, before any CUDA call, for sizes out of range, a NULL pointer (with P > 0) or an overlap.
 * Stream-ordered without host sync; every result is bitwise reproducible. */
size_t f3dgs_knn_graph_scratch_bytes(int P, int k);
int f3dgs_knn_graph(int P, int k, const float* points, int32_t* idx, float* dist2, int32_t* order, char* scratch,
                    void* cuda_stream);
int f3dgs_knn_reverse(int P, int k, const int32_t* idx, int32_t* offsets, int32_t* sources, char* scratch,
                      void* cuda_stream);
int f3dgs_feature_tv_accum(int P, int k, int C, const float* features, const int32_t* idx, const int32_t* offsets,
                           const int32_t* sources, const int32_t* order, double weight, long long n_edges, float* grad,
                           double* loss, void* cuda_stream);
int f3dgs_feature_fill(int P, int k, int C, const float* features, const float* weights, const int32_t* idx,
                       float min_weight, float* out, void* cuda_stream);

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
