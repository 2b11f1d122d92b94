/*
 * oracle/f3dgs_oracle.c -- CPU restatement of the reference rasterizer's algorithm.
 *
 * TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs.  Nothing on the product path links or calls this file.
 *
 * The reference has no CPU implementation (SURVEY.md section 0); this is a plain-C restatement of its
 * CUDA algorithm, function by function, each citing the reference file:line it follows
 * (DGR = <reference checkout>/submodules/diff-gaussian-rasterization-feature).  Pinning: the reference
 * ships no golden vectors, so the oracle is pinned against outputs of the reference extension
 * itself (oracle/_ref, built from the unmodified sources by oracle/build_ref.py and run on the
 * GPU by oracle/make_golden.py); the vectors are committed under tests/golden/.
 *
 * Numerics: the forward per-Gaussian stage reproduces the exact fp32 operation sequence of the
 * reference's build (FMA placement read off its PTX *and* SASS -- ptxas fuses further
 * mul/add pairs the PTX still shows separately; fmaf() here, -ffp-contract=off), so radii / tile
 * rectangles / depth keys / point_list / ranges are bit-identical to the GPU.
 * expf() comes from libm and differs from CUDA's by <= 2 ulp, so images agree to ~1e-6 and
 * n_contrib can differ on measure-zero threshold ties.
 *
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -mavx2 -shared -fPIC (see oracle/__init__.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define TILE 16

static inline float dot3r(float a0, float b0, float a1, float b1, float a2, float b2) {
    /* a0*b0 + a1*b1 + a2*b2 as nvcc contracts it: middle product plain, outer two fused */
    return fmaf(a2, b2, fmaf(a0, b0, a1 * b1));
}
/* DGR/cuda_rasterizer/auxiliary.h:58-77 transformPoint4x3 / 4x4, one row */
static inline float xform_row(const float* m, int r, float x, float y, float z) {
    return m[12 + r] + fmaf(z, m[8 + r], fmaf(x, m[r], y * m[4 + r]));
}
/* auxiliary.h:41-44 ndc2Pix (double arithmetic because of the unsuffixed literals) */
static inline float ndc2pix(float v, int S) { return (float)(fma((double)v + 1.0, (double)S, -1.0) * 0.5); }

static inline int imax(int a, int b) { return a > b ? a : b; }
static inline uint32_t umin(uint32_t a, uint32_t b) { return a < b ? a : b; }

/* auxiliary.h:46-56 getRect */
static inline void get_rect(float px, float py, int radius, uint32_t gx, uint32_t gy, uint32_t* x0, uint32_t* y0,
                            uint32_t* x1, uint32_t* y1) {
    const float rf = (float)radius;
    *x0 = umin(gx, (uint32_t)imax(0, (int)((px - rf) * 0.0625f)));
    *y0 = umin(gy, (uint32_t)imax(0, (int)((py - rf) * 0.0625f)));
    *x1 = umin(gx, (uint32_t)imax(0, (int)((((px + rf) + 16.0f) + -1.0f) * 0.0625f)));
    *y1 = umin(gy, (uint32_t)imax(0, (int)((((py + rf) + 16.0f) + -1.0f) * 0.0625f)));
}

static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                               -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

/* DGR/cuda_rasterizer/forward.cu:20-72 computeColorFromSH */
static void sh_to_rgb(int deg, const float* sh, const float* p, const float* cam, float* rgb, uint8_t* clamped) {
    const float dx = p[0] - cam[0], dy = p[1] - cam[1], dz = p[2] - cam[2];
    const float len = sqrtf(dot3r(dx, dx, dy, dy, dz, dz));
    const float x = dx / len, y = dy / len, z = dz / len;
    float res[3];
    for (int c = 0; c < 3; c++) res[c] = sh[c] * SH_C0;
    if (deg > 0) {
        const float ty = y * SH_C1, tz = z * SH_C1, tx = x * SH_C1;
        for (int c = 0; c < 3; c++) {
            float r = fmaf(-ty, sh[3 + c], res[c]); /* ptxas fuses res - ty*sh (SASS: FFMA -R, R, R) */
            r = fmaf(tz, sh[6 + c], r);
            res[c] = fmaf(-tx, sh[9 + c], r);
        }
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            const float zz2 = zz + zz;
            const float k4 = xy * SH_C2[0], k5 = yz * SH_C2[1], k6 = ((zz2 - xx) - yy) * SH_C2[2];
            const float k7 = xz * SH_C2[3], xxmyy = xx - yy, k8 = xxmyy * SH_C2[4];
            for (int c = 0; c < 3; c++) {
                float r = fmaf(k4, sh[12 + c], res[c]);
                r = fmaf(k5, sh[15 + c], r);
                r = fmaf(k6, sh[18 + c], r);
                r = fmaf(k7, sh[21 + c], r);
                res[c] = fmaf(k8, sh[24 + c], r);
            }
            if (deg > 2) {
                /* SASS: the x3 / x4 products are fused into the subtractions that consume them */
                const float k9 = (y * SH_C3[0]) * fmaf(xx, 3.0f, -yy);
                const float k10 = z * (xy * SH_C3[1]);
                const float q = fmaf(zz, 4.0f, -xx) - yy;
                const float k11 = (y * SH_C3[2]) * q;
                const float k12 = (z * SH_C3[3]) * fmaf(yy, -3.0f, fmaf(xx, -3.0f, zz2));
                const float k13 = (x * SH_C3[4]) * q;
                const float k14 = (z * SH_C3[5]) * xxmyy;
                const float k15 = (x * SH_C3[6]) * fmaf(yy, -3.0f, xx);
                for (int c = 0; c < 3; c++) {
                    float r = fmaf(k9, sh[27 + c], res[c]);
                    r = fmaf(k10, sh[30 + c], r);
                    r = fmaf(k11, sh[33 + c], r);
                    r = fmaf(k12, sh[36 + c], r);
                    r = fmaf(k13, sh[39 + c], r);
                    r = fmaf(k14, sh[42 + c], r);
                    res[c] = fmaf(k15, sh[45 + c], r);
                }
            }
        }
    }
    for (int c = 0; c < 3; c++) {
        float v = res[c] + 0.5f;
        clamped[c] = (v < 0.f);
        rgb[c] = v < 0.f ? 0.f : v;
    }
}

/* forward.cu:119-153 computeCov3D */
static void cov3d_from_scale_rot(const float* s3, float mod, const float* q4, float* cov) {
    const float sx = mod * s3[0], sy = mod * s3[1], sz = mod * s3[2];
    const float r = q4[0], x = q4[1], y = q4[2], z = q4[3];
    /* SASS of the reference build: of each product pair (xy,rz) (xz,ry) (yz,rx) ptxas keeps one product as a
     * rounded FMUL and fuses the other into both the sum and the difference */
    const float yy = y * y, zz = z * z, rz = r * z, xz = x * z, rx = r * x;
    const float a = yy + zz, b = fmaf(x, x, zz), c = fmaf(x, x, yy);
    const float R00 = 1.0f - (a + a), R11 = 1.0f - (b + b), R22 = 1.0f - (c + c);
    float t;
    const float m00 = sx * R00;
    t = fmaf(x, y, -rz); const float m01 = sy * (t + t);  /* 2(xy - rz) */
    t = fmaf(r, y, xz);  const float m02 = sz * (t + t);  /* 2(xz + ry) */
    t = fmaf(x, y, rz);  const float m10 = sx * (t + t);  /* 2(xy + rz) */
    const float m11 = sy * R11;
    t = fmaf(y, z, -rx); const float m12 = sz * (t + t);  /* 2(yz - rx) */
    t = fmaf(-r, y, xz); const float m20 = sx * (t + t);  /* 2(xz - ry) */
    t = fmaf(y, z, rx);  const float m21 = sy * (t + t);  /* 2(yz + rx) */
    const float m22 = sz * R22;
    cov[0] = dot3r(m00, m00, m01, m01, m02, m02);
    cov[1] = dot3r(m10, m00, m11, m01, m12, m02);
    cov[2] = dot3r(m20, m00, m21, m01, m22, m02);
    cov[3] = dot3r(m10, m10, m11, m11, m12, m12);
    cov[4] = dot3r(m20, m10, m21, m11, m22, m12);
    cov[5] = dot3r(m20, m20, m21, m21, m22, m22);
}

typedef struct {
    float a, b, c;
    float T[2][3];
    float tx, ty, tz, txtz, tytz;
} cov2d_t;

/* forward.cu:75-114 computeCov2D (returns cov with the 0.3 dilation) */
static cov2d_t project_cov(const float* p, const float* vm, float fx, float fy, float tanx, float tany,
                           const float* cv) {
    cov2d_t o;
    const float tx = xform_row(vm, 0, p[0], p[1], p[2]);
    const float ty = xform_row(vm, 1, p[0], p[1], p[2]);
    const float tz = xform_row(vm, 2, p[0], p[1], p[2]);
    const float limx = tanx * 1.3f, limy = tany * 1.3f;
    o.txtz = tx / tz;
    o.tytz = ty / tz;
    const float cx = fminf(limx, fmaxf(-limx, o.txtz));
    const float cy = fminf(limy, fmaxf(-limy, o.tytz));
    const float ntz = -tz, tz2 = tz * tz;
    const float J00 = fx / tz, J02 = (fx * (cx * ntz)) / tz2;
    const float J11 = fy / tz, J12 = (fy * (cy * ntz)) / tz2;
    o.tx = cx * tz; o.ty = cy * tz; o.tz = tz;
    o.T[0][0] = fmaf(vm[2], J02, vm[0] * J00);
    o.T[0][1] = fmaf(vm[6], J02, vm[4] * J00);
    o.T[0][2] = fmaf(J02, vm[10], vm[8] * J00);
    o.T[1][0] = fmaf(vm[2], J12, J11 * vm[1]);
    o.T[1][1] = fmaf(vm[6], J12, J11 * vm[5]);
    o.T[1][2] = fmaf(J12, vm[10], J11 * vm[9]);
    const float* T0 = o.T[0];
    const float* T1 = o.T[1];
    const float A00 = dot3r(T0[0], cv[0], T0[1], cv[1], T0[2], cv[2]);
    const float A10 = dot3r(T1[0], cv[0], T1[1], cv[1], T1[2], cv[2]);
    const float A01 = dot3r(T0[0], cv[1], T0[1], cv[3], T0[2], cv[4]);
    const float A11 = dot3r(T1[0], cv[1], T1[1], cv[3], T1[2], cv[4]);
    const float A02 = dot3r(T0[0], cv[2], T0[1], cv[4], T0[2], cv[5]);
    const float A12 = dot3r(T1[0], cv[2], T1[1], cv[4], T1[2], cv[5]);
    o.a = dot3r(T0[0], A00, T0[1], A01, T0[2], A02) + 0.3f;
    o.b = dot3r(T0[0], A10, T0[1], A11, T0[2], A12);
    o.c = dot3r(T1[0], A10, T1[1], A11, T1[2], A12) + 0.3f;
    return o;
}

/* ------------------------------------------------------------------------------------------
 * FORWARD::preprocessCUDA, forward.cu:156-256 (+ in_frustum auxiliary.h:145-170).
 * Outputs are the reference's GeometryState fields (rasterizer_impl.cu:154-170).
 * Returns sum(tiles_touched) = num_rendered.
 */
long long oracle_preprocess(int P, int D, int M, const float* means3D, const float* scales, float scale_modifier,
                            const float* rotations, const float* opacities, const float* shs,
                            const float* cov3D_precomp, const float* colors_precomp, const float* viewmatrix,
                            const float* projmatrix, const float* cam_pos, int W, int H, float tan_fovx,
                            float tan_fovy, int* radii, float* means2D, float* depths, float* cov3Ds, float* rgb,
                            float* conic_opacity, uint8_t* clamped, uint32_t* tiles_touched) {
    const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx); /* rasterizer_impl.cu:225-226 */
    const uint32_t gx = (uint32_t)((W + TILE - 1) / TILE), gy = (uint32_t)((H + TILE - 1) / TILE);
    long long total = 0;
#pragma omp parallel for schedule(static) reduction(+ : total)
    for (int idx = 0; idx < P; idx++) {
        radii[idx] = 0;
        tiles_touched[idx] = 0;
        const float* p = means3D + 3 * idx;
        const float depth = xform_row(viewmatrix, 2, p[0], p[1], p[2]);
        if (depth <= 0.2f) continue; /* auxiliary.h:160 */
        const float hx = xform_row(projmatrix, 0, p[0], p[1], p[2]);
        const float hy = xform_row(projmatrix, 1, p[0], p[1], p[2]);
        const float hw = xform_row(projmatrix, 3, p[0], p[1], p[2]);
        const float p_w = 1.0f / (hw + 0.0000001f);
        const float projx = hx * p_w, projy = hy * p_w;
        float cvbuf[6];
        const float* cv;
        if (cov3D_precomp) {
            cv = cov3D_precomp + 6 * idx;
        } else {
            cov3d_from_scale_rot(scales + 3 * idx, scale_modifier, rotations + 4 * idx, cvbuf);
            memcpy(cov3Ds + 6 * idx, cvbuf, sizeof(cvbuf));
            cv = cvbuf;
        }
        const cov2d_t c2 = project_cov(p, viewmatrix, focal_x, focal_y, tan_fovx, tan_fovy, cv);
        const float det = fmaf(c2.a, c2.c, -(c2.b * c2.b)); /* SASS: FMUL b*b; FFMA a, c, -bb */
        if (det == 0.0f) continue;
        const float det_inv = 1.0f / det;
        const float conA = c2.c * det_inv, conB = det_inv * -c2.b, conC = c2.a * det_inv;
        const float mid = (c2.a + c2.c) * 0.5f;
        const float sq = sqrtf(fmaxf(fmaf(mid, mid, -det), 0.1f)); /* SASS: FFMA mid, mid, -det */
        const float lam = fmaxf(mid + sq, mid - sq);
        const float rad_f = ceilf(sqrtf(lam) * 3.0f);
        const int rad = (int)rad_f;
        const float ix = ndc2pix(projx, W), iy = ndc2pix(projy, H);
        uint32_t x0, y0, x1, y1;
        get_rect(ix, iy, rad, gx, gy, &x0, &y0, &x1, &y1);
        const uint32_t area = (x1 - x0) * (y1 - y0);
        if (area == 0) continue;
        if (!colors_precomp) {
            sh_to_rgb(D, shs + (size_t)idx * M * 3, p, cam_pos, rgb + 3 * idx, clamped + 3 * idx);
        }
        depths[idx] = depth;
        radii[idx] = rad;
        means2D[2 * idx] = ix;
        means2D[2 * idx + 1] = iy;
        conic_opacity[4 * idx] = conA;
        conic_opacity[4 * idx + 1] = conB;
        conic_opacity[4 * idx + 2] = conC;
        conic_opacity[4 * idx + 3] = opacities[idx];
        tiles_touched[idx] = area;
        total += area;
    }
    return total;
}

/* ------------------------------------------------------------------------------------------
 * Binning: InclusiveSum + duplicateWithKeys (rasterizer_impl.cu:70-111) + stable radix sort on
 * (tile << 32 | depth bits) (rasterizer_impl.cu:305-310) + identifyTileRanges (:116-138).
 * keys/point_list have R entries; ranges has 2 * tiles entries (zero-initialised here, :312).
 */
void oracle_bin(int P, long long R, const int* radii, const float* means2D, const float* depths,
                const uint32_t* tiles_touched, int W, int H, uint64_t* keys_sorted, uint32_t* point_list,
                uint32_t* ranges) {
    const uint32_t gx = (uint32_t)((W + TILE - 1) / TILE), gy = (uint32_t)((H + TILE - 1) / TILE);
    const size_t tiles = (size_t)gx * gy;
    memset(ranges, 0, tiles * 2 * sizeof(uint32_t));
    if (R <= 0) return;
    uint64_t* k0 = (uint64_t*)malloc((size_t)R * 8);
    uint64_t* k1 = (uint64_t*)malloc((size_t)R * 8);
    uint32_t* v0 = (uint32_t*)malloc((size_t)R * 4);
    uint32_t* v1 = (uint32_t*)malloc((size_t)R * 4);
    size_t off = 0;
    for (int idx = 0; idx < P; idx++) {
        if (radii[idx] > 0) {
            uint32_t x0, y0, x1, y1;
            get_rect(means2D[2 * idx], means2D[2 * idx + 1], radii[idx], gx, gy, &x0, &y0, &x1, &y1);
            uint32_t dbits;
            memcpy(&dbits, depths + idx, 4);
            for (uint32_t y = y0; y < y1; y++)
                for (uint32_t x = x0; x < x1; x++) {
                    k0[off] = ((uint64_t)(y * gx + x) << 32) | dbits;
                    v0[off] = (uint32_t)idx;
                    off++;
                }
        }
        (void)tiles_touched;
    }
    /* stable LSD radix sort, 8 bits per pass over all 64 key bits (a superset of the reference's
     * [0, 32+bit) window: the bits above are zero, so the order is identical) */
    for (int pass = 0; pass < 8; pass++) {
        size_t hist[257];
        memset(hist, 0, sizeof(hist));
        const int sh = pass * 8;
        for (long long i = 0; i < R; i++) hist[((k0[i] >> sh) & 0xFF) + 1]++;
        for (int b = 0; b < 256; b++) hist[b + 1] += hist[b];
        for (long long i = 0; i < R; i++) {
            const size_t d = hist[(k0[i] >> sh) & 0xFF]++;
            k1[d] = k0[i];
            v1[d] = v0[i];
        }
        uint64_t* tk = k0; k0 = k1; k1 = tk;
        uint32_t* tv = v0; v0 = v1; v1 = tv;
    }
    memcpy(keys_sorted, k0, (size_t)R * 8);
    memcpy(point_list, v0, (size_t)R * 4);
    for (long long i = 0; i < R; i++) {
        const uint32_t cur = (uint32_t)(k0[i] >> 32);
        if (i == 0) {
            ranges[2 * cur] = 0;
        } else {
            const uint32_t prev = (uint32_t)(k0[i - 1] >> 32);
            if (cur != prev) {
                ranges[2 * prev + 1] = (uint32_t)i;
                ranges[2 * cur] = (uint32_t)i;
            }
        }
        if (i == R - 1) ranges[2 * cur + 1] = (uint32_t)R;
    }
    free(k0); free(k1); free(v0); free(v1);
}

/* ------------------------------------------------------------------------------------------
 * forward renderCUDA<3>, forward.cu:261-396.  colors = rgb from SH or colors_precomp
 * (rasterizer_impl.cu:323).  tile_begin/tile_end restrict the tiles processed (bench sampling).
 */
void oracle_render(int W, int H, int C, const uint32_t* ranges, const uint32_t* point_list, const float* means2D,
                   const float* colors, const float* features, const float* depths, const float* conic_opacity,
                   const float* bg, float* final_T, uint32_t* n_contrib, float* out_color, float* out_feature,
                   float* out_depth, int tile_begin, int tile_end) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    const size_t HW = (size_t)H * W;
    if (tile_end < 0 || tile_end > gx * gy) tile_end = gx * gy;
#pragma omp parallel
    {
        float* SF = (float*)malloc(sizeof(float) * (C > 0 ? C : 1));
#pragma omp for schedule(dynamic, 1)
        for (int tile = tile_begin; tile < tile_end; tile++) {
            const int tyi = tile / gx, txi = tile % gx;
            const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
            for (int ly = 0; ly < TILE; ly++)
                for (int lx = 0; lx < TILE; lx++) {
                    const int px = txi * TILE + lx, py = tyi * TILE + ly;
                    if (px >= W || py >= H) continue;
                    const size_t pix = (size_t)py * W + px;
                    const float pxf = (float)px, pyf = (float)py;
                    float T = 1.0f, Cc[3] = {0, 0, 0}, Dp = 0.f;
                    uint32_t contributor = 0, last = 0;
                    for (int c = 0; c < C; c++) SF[c] = 0.f;
                    for (uint32_t i = r0; i < r1; i++) {
                        contributor++;
                        const uint32_t g = point_list[i];
                        const float dx = means2D[2 * g] - pxf, dy = means2D[2 * g + 1] - pyf;
                        const float* co = conic_opacity + 4 * g;
                        const float t4 = fmaf(dx, dx * co[0], dy * (dy * co[2]));
                        const float power = fmaf(t4, -0.5f, -(dy * (dx * co[1]))); /* SASS: FFMA t4, -0.5, -R */
                        if (power > 0.0f) continue;
                        const float alpha = fminf(co[3] * expf(power), 0.99f);
                        if (alpha < 1.0f / 255.0f) continue;
                        const float test_T = T * (1.0f - alpha);
                        if (test_T < 0.0001f) break; /* done = true: the Gaussian is NOT blended */
                        for (int ch = 0; ch < 3; ch++) Cc[ch] = fmaf(T, alpha * colors[3 * g + ch], Cc[ch]);
                        const float w = T * alpha;
                        Dp = fmaf(w, depths[g], Dp);
                        const float* f = features + (size_t)g * C;
                        for (int ch = 0; ch < C; ch++) SF[ch] = fmaf(T, alpha * f[ch], SF[ch]);
                        T = test_T;
                        last = contributor;
                    }
                    final_T[pix] = T;
                    n_contrib[pix] = last;
                    for (int ch = 0; ch < 3; ch++) out_color[ch * HW + pix] = fmaf(T, bg[ch], Cc[ch]);
                    out_depth[pix] = Dp;
                    for (int ch = 0; ch < C; ch++) out_feature[ch * HW + pix] = SF[ch];
                }
        }
        free(SF);
    }
}

static inline void atomic_addf(float* p, float v, int par) {
    if (par) {
#pragma omp atomic
        *p += v;
    } else {
        *p += v;
    }
}

/* ------------------------------------------------------------------------------------------
 * backward renderCUDA<3>, backward.cu:407-620.  Gradients are accumulated (+=) into zeroed
 * arrays, as the reference's atomicAdd into torch::zeros tensors.  With one thread the result
 * is deterministic (pixel-major order); with more threads float atomics are used.
 */
void oracle_render_backward(int W, int H, int C, const uint32_t* ranges, const uint32_t* point_list,
                            const float* bg, const float* means2D, const float* conic_opacity, const float* colors,
                            const float* depths, const float* final_T, const uint32_t* n_contrib,
                            const float* dL_dpix, const float* dL_dfeat_pix, const float* dL_ddepth,
                            float* dL_dmean2D /*[P,3]*/, float* dL_dconic /*[P,4]*/, float* dL_dopacity,
                            float* dL_dcolor /*[P,3]*/, float* dL_dfeature /*[P,C]*/, float* dL_dz, int tile_begin,
                            int tile_end) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    const size_t HW = (size_t)H * W;
    if (tile_end < 0 || tile_end > gx * gy) tile_end = gx * gy;
    int par = 0;
#ifdef _OPENMP
    par = omp_get_max_threads() > 1;
#endif
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;
#pragma omp parallel
    {
        float* dLf = (float*)malloc(sizeof(float) * (C > 0 ? C : 1));
#pragma omp for schedule(dynamic, 1)
        for (int tile = tile_begin; tile < tile_end; tile++) {
            const int tyi = tile / gx, txi = tile % gx;
            const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
            for (int ly = 0; ly < TILE; ly++)
                for (int lx = 0; lx < TILE; lx++) {
                    const int px = txi * TILE + lx, py = tyi * TILE + ly;
                    if (px >= W || py >= H) continue;
                    const size_t pix = (size_t)py * W + px;
                    const float pxf = (float)px, pyf = (float)py;
                    const float T_final = final_T[pix];
                    float T = T_final;
                    const uint32_t last_contributor = n_contrib[pix];
                    uint32_t contributor = r1 - r0;
                    float accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0};
                    float last_alpha = 0.f, accum_depth_rec = 0.f, last_depth = 0.f;
                    float dLp[3];
                    for (int ch = 0; ch < 3; ch++) dLp[ch] = dL_dpix[ch * HW + pix];
                    const float dLd = dL_ddepth[pix];
                    for (int ch = 0; ch < C; ch++) dLf[ch] = dL_dfeat_pix[ch * HW + pix];
                    float bg_dot = 0.f;
                    for (int ch = 0; ch < 3; ch++) bg_dot += bg[ch] * dLp[ch];
                    for (uint32_t i = r1; i-- > r0;) {
                        contributor--;
                        if (contributor >= last_contributor) continue;
                        const uint32_t g = point_list[i];
                        const float dx = means2D[2 * g] - pxf, dy = means2D[2 * g + 1] - pyf;
                        const float* co = conic_opacity + 4 * g;
                        const float t4 = fmaf(dx, dx * co[0], dy * (dy * co[2]));
                        const float power = fmaf(t4, -0.5f, -(dy * (dx * co[1]))); /* SASS: FFMA t4, -0.5, -R */
                        if (power > 0.0f) continue;
                        const float G = expf(power);
                        const float alpha = fminf(co[3] * G, 0.99f);
                        if (alpha < 1.0f / 255.0f) continue;
                        T = T / (1.f - alpha);
                        const float w = alpha * T;
                        float dL_dalpha = 0.f;
                        for (int ch = 0; ch < 3; ch++) {
                            const float c = colors[3 * g + ch];
                            accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
                            last_color[ch] = c;
                            dL_dalpha += (c - accum_rec[ch]) * dLp[ch];
                            atomic_addf(dL_dcolor + 3 * g + ch, w * dLp[ch], par);
                        }
                        const float c_d = depths[g];
                        accum_depth_rec = last_alpha * last_depth + (1.f - last_alpha) * accum_depth_rec;
                        last_depth = c_d;
                        dL_dalpha += (c_d - accum_depth_rec) * dLd;
                        /* features feed dL_dsemantic_feature only: backward.cu:575 is commented out */
                        float* gf = dL_dfeature + (size_t)g * C;
                        for (int ch = 0; ch < C; ch++) atomic_addf(gf + ch, w * dLf[ch], par);
                        dL_dalpha *= T;
                        last_alpha = alpha;
                        dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
                        const float dL_dG = co[3] * dL_dalpha;
                        const float gdx = G * dx, gdy = G * dy;
                        const float dG_ddelx = -gdx * co[0] - gdy * co[1];
                        const float dG_ddely = -gdy * co[2] - gdx * co[1];
                        atomic_addf(dL_dmean2D + 3 * g, dL_dG * dG_ddelx * ddelx_dx, par);
                        atomic_addf(dL_dmean2D + 3 * g + 1, dL_dG * dG_ddely * ddely_dy, par);
                        atomic_addf(dL_dconic + 4 * g, -0.5f * gdx * dx * dL_dG, par);
                        atomic_addf(dL_dconic + 4 * g + 1, -0.5f * gdx * dy * dL_dG, par);
                        atomic_addf(dL_dconic + 4 * g + 3, -0.5f * gdy * dy * dL_dG, par);
                        atomic_addf(dL_dopacity + g, G * dL_dalpha, par);
                        atomic_addf(dL_dz + g, w * dLd, par);
                    }
                }
        }
        free(dLf);
    }
}

/* auxiliary.h:107-117 dnormvdv (float3) */
static void dnormvdv3(const float* v, const float* dv, float* o) {
    const float sum2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    const float inv = 1.0f / sqrtf(sum2 * sum2 * sum2);
    o[0] = ((+sum2 - v[0] * v[0]) * dv[0] - v[1] * v[0] * dv[1] - v[2] * v[0] * dv[2]) * inv;
    o[1] = (-v[0] * v[1] * dv[0] + (sum2 - v[1] * v[1]) * dv[1] - v[2] * v[1] * dv[2]) * inv;
    o[2] = (-v[0] * v[2] * dv[0] - v[1] * v[2] * dv[1] + (sum2 - v[2] * v[2]) * dv[2]) * inv;
}

/* ------------------------------------------------------------------------------------------
 * computeCov2DCUDA (backward.cu:144-274) followed by BACKWARD::preprocessCUDA (:346-404) with
 * computeColorFromSH backward (:20-139) and computeCov3D backward (:278-341).
 * `clamped` is the [P,3] flag array of the forward.  Outputs must be zero-initialised.
 */
void oracle_preprocess_backward(int P, int D, int M, const float* means3D, const int* radii, const float* shs,
                                const uint8_t* clamped, const float* scales, const float* rotations,
                                float scale_modifier, const float* cov3Ds, const float* viewmatrix,
                                const float* projmatrix, const float* cam_pos, int W, int H, float tan_fovx,
                                float tan_fovy, const float* dL_dmean2D, const float* dL_dconic,
                                const float* dL_dcolor, const float* dL_dz, float* dL_dmean3D, float* dL_dcov3D,
                                float* dL_dsh, float* dL_dscale, float* dL_drot) {
    const float h_y = H / (2.0f * tan_fovy), h_x = W / (2.0f * tan_fovx);
    const float* vm = viewmatrix;
    const float* proj = projmatrix;
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < P; idx++) {
        if (!(radii[idx] > 0)) continue;
        const float* m = means3D + 3 * idx;
        const float* cv = cov3Ds + 6 * idx;
        const cov2d_t c2 = project_cov(m, vm, h_x, h_y, tan_fovx, tan_fovy, cv);
        const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
        const float x_grad_mul = (c2.txtz < -limx || c2.txtz > limx) ? 0.f : 1.f;
        const float y_grad_mul = (c2.tytz < -limy || c2.tytz > limy) ? 0.f : 1.f;
        const float a = c2.a, b = c2.b, c = c2.c;
        const float dLcx = dL_dconic[4 * idx], dLcy = dL_dconic[4 * idx + 1], dLcz = dL_dconic[4 * idx + 3];
        const float denom = a * c - b * b;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        float dL_da = 0, dL_db = 0, dL_dc = 0;
        const float(*T)[3] = c2.T; /* T[c][r] as GLM indexes it */
        float dcov[6] = {0, 0, 0, 0, 0, 0};
        if (denom2inv != 0) {
            dL_da = denom2inv * (-c * c * dLcx + 2 * b * c * dLcy + (denom - a * c) * dLcz);
            dL_dc = denom2inv * (-a * a * dLcz + 2 * a * b * dLcy + (denom - a * c) * dLcx);
            dL_db = denom2inv * 2 * (b * c * dLcx - (denom + 2 * b * b) * dLcy + a * b * dLcz);
            dcov[0] = (T[0][0] * T[0][0] * dL_da + T[0][0] * T[1][0] * dL_db + T[1][0] * T[1][0] * dL_dc);
            dcov[3] = (T[0][1] * T[0][1] * dL_da + T[0][1] * T[1][1] * dL_db + T[1][1] * T[1][1] * dL_dc);
            dcov[5] = (T[0][2] * T[0][2] * dL_da + T[0][2] * T[1][2] * dL_db + T[1][2] * T[1][2] * dL_dc);
            dcov[1] = 2 * T[0][0] * T[0][1] * dL_da + (T[0][0] * T[1][1] + T[0][1] * T[1][0]) * dL_db +
                      2 * T[1][0] * T[1][1] * dL_dc;
            dcov[2] = 2 * T[0][0] * T[0][2] * dL_da + (T[0][0] * T[1][2] + T[0][2] * T[1][0]) * dL_db +
                      2 * T[1][0] * T[1][2] * dL_dc;
            dcov[4] = 2 * T[0][2] * T[0][1] * dL_da + (T[0][1] * T[1][2] + T[0][2] * T[1][1]) * dL_db +
                      2 * T[1][1] * T[1][2] * dL_dc;
        }
        for (int i = 0; i < 6; i++) dL_dcov3D[6 * idx + i] = dcov[i];
        const float V[3][3] = {{cv[0], cv[1], cv[2]}, {cv[1], cv[3], cv[4]}, {cv[2], cv[4], cv[5]}};
        float dT[2][3];
        for (int j = 0; j < 3; j++) {
            const float t0 = T[0][0] * V[j][0] + T[0][1] * V[j][1] + T[0][2] * V[j][2];
            const float t1 = T[1][0] * V[j][0] + T[1][1] * V[j][1] + T[1][2] * V[j][2];
            dT[0][j] = 2 * t0 * dL_da + t1 * dL_db;
            dT[1][j] = 2 * t1 * dL_dc + t0 * dL_db;
        }
        const float dL_dJ00 = vm[0] * dT[0][0] + vm[4] * dT[0][1] + vm[8] * dT[0][2];
        const float dL_dJ02 = vm[2] * dT[0][0] + vm[6] * dT[0][1] + vm[10] * dT[0][2];
        const float dL_dJ11 = vm[1] * dT[1][0] + vm[5] * dT[1][1] + vm[9] * dT[1][2];
        const float dL_dJ12 = vm[2] * dT[1][0] + vm[6] * dT[1][1] + vm[10] * dT[1][2];
        const float tz = 1.f / c2.tz, tz2 = tz * tz, tz3 = tz2 * tz;
        const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
        const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
        const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * c2.tx) * tz3 * dL_dJ02 +
                             (2 * h_y * c2.ty) * tz3 * dL_dJ12;
        float g[3];
        g[0] = vm[0] * dL_dtx + vm[1] * dL_dty + vm[2] * dL_dtz;
        g[1] = vm[4] * dL_dtx + vm[5] * dL_dty + vm[6] * dL_dtz;
        g[2] = vm[8] * dL_dtx + vm[9] * dL_dty + vm[10] * dL_dtz;
        {
            const float hw = proj[3] * m[0] + proj[7] * m[1] + proj[11] * m[2] + proj[15];
            const float m_w = 1.0f / (hw + 0.0000001f);
            const float mul1 = (proj[0] * m[0] + proj[4] * m[1] + proj[8] * m[2] + proj[12]) * m_w * m_w;
            const float mul2 = (proj[1] * m[0] + proj[5] * m[1] + proj[9] * m[2] + proj[13]) * m_w * m_w;
            const float d2x = dL_dmean2D[3 * idx], d2y = dL_dmean2D[3 * idx + 1];
            float ax = (proj[0] * m_w - proj[3] * mul1) * d2x + (proj[1] * m_w - proj[3] * mul2) * d2y;
            float ay = (proj[4] * m_w - proj[7] * mul1) * d2x + (proj[5] * m_w - proj[7] * mul2) * d2y;
            float az = (proj[8] * m_w - proj[11] * mul1) * d2x + (proj[9] * m_w - proj[11] * mul2) * d2y;
            const float dldz = dL_dz[idx];
            ax += dldz * vm[2];
            ay += dldz * vm[6];
            az += dldz * vm[10];
            g[0] += ax; g[1] += ay; g[2] += az;
        }
        if (shs) {
            const float* sh = shs + (size_t)idx * M * 3;
            float* dsh = dL_dsh + (size_t)idx * M * 3;
            const float dir_orig[3] = {m[0] - cam_pos[0], m[1] - cam_pos[1], m[2] - cam_pos[2]};
            const float il = 1.0f / sqrtf(dir_orig[0] * dir_orig[0] + dir_orig[1] * dir_orig[1] + dir_orig[2] * dir_orig[2]);
            const float x = dir_orig[0] * il, y = dir_orig[1] * il, z = dir_orig[2] * il;
            float dRGB[3];
            for (int ch = 0; ch < 3; ch++) dRGB[ch] = clamped[3 * idx + ch] ? 0.f : dL_dcolor[3 * idx + ch];
            float dx_[3] = {0, 0, 0}, dy_[3] = {0, 0, 0}, dz_[3] = {0, 0, 0};
#define SHC(k, c) sh[3 * (k) + (c)]
#define WR(k, coef) do { const float cf_ = (coef); for (int c_ = 0; c_ < 3; c_++) dsh[3 * (k) + c_] = cf_ * dRGB[c_]; } while (0)
            WR(0, SH_C0);
            if (D > 0) {
                WR(1, -SH_C1 * y); WR(2, SH_C1 * z); WR(3, -SH_C1 * x);
                for (int ch = 0; ch < 3; ch++) {
                    dx_[ch] = -SH_C1 * SHC(3, ch); dy_[ch] = -SH_C1 * SHC(1, ch); dz_[ch] = SH_C1 * SHC(2, ch);
                }
                if (D > 1) {
                    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    WR(4, SH_C2[0] * xy); WR(5, SH_C2[1] * yz); WR(6, SH_C2[2] * (2.f * zz - xx - yy));
                    WR(7, SH_C2[3] * xz); WR(8, SH_C2[4] * (xx - yy));
                    for (int ch = 0; ch < 3; ch++) {
                        dx_[ch] += SH_C2[0] * y * SHC(4, ch) + SH_C2[2] * 2.f * -x * SHC(6, ch) + SH_C2[3] * z * SHC(7, ch) + SH_C2[4] * 2.f * x * SHC(8, ch);
                        dy_[ch] += SH_C2[0] * x * SHC(4, ch) + SH_C2[1] * z * SHC(5, ch) + SH_C2[2] * 2.f * -y * SHC(6, ch) + SH_C2[4] * 2.f * -y * SHC(8, ch);
                        dz_[ch] += SH_C2[1] * y * SHC(5, ch) + SH_C2[2] * 2.f * 2.f * z * SHC(6, ch) + SH_C2[3] * x * SHC(7, ch);
                    }
                    if (D > 2) {
                        WR(9, SH_C3[0] * y * (3.f * xx - yy)); WR(10, SH_C3[1] * xy * z);
                        WR(11, SH_C3[2] * y * (4.f * zz - xx - yy)); WR(12, SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy));
                        WR(13, SH_C3[4] * x * (4.f * zz - xx - yy)); WR(14, SH_C3[5] * z * (xx - yy));
                        WR(15, SH_C3[6] * x * (xx - 3.f * yy));
                        for (int ch = 0; ch < 3; ch++) {
                            dx_[ch] += (SH_C3[0] * SHC(9, ch) * 3.f * 2.f * xy + SH_C3[1] * SHC(10, ch) * yz + SH_C3[2] * SHC(11, ch) * -2.f * xy +
                                        SH_C3[3] * SHC(12, ch) * -3.f * 2.f * xz + SH_C3[4] * SHC(13, ch) * (-3.f * xx + 4.f * zz - yy) +
                                        SH_C3[5] * SHC(14, ch) * 2.f * xz + SH_C3[6] * SHC(15, ch) * 3.f * (xx - yy));
                            dy_[ch] += (SH_C3[0] * SHC(9, ch) * 3.f * (xx - yy) + SH_C3[1] * SHC(10, ch) * xz + SH_C3[2] * SHC(11, ch) * (-3.f * yy + 4.f * zz - xx) +
                                        SH_C3[3] * SHC(12, ch) * -3.f * 2.f * yz + SH_C3[4] * SHC(13, ch) * -2.f * xy +
                                        SH_C3[5] * SHC(14, ch) * -2.f * yz + SH_C3[6] * SHC(15, ch) * -3.f * 2.f * xy);
                            dz_[ch] += (SH_C3[1] * SHC(10, ch) * xy + SH_C3[2] * SHC(11, ch) * 4.f * 2.f * yz + SH_C3[3] * SHC(12, ch) * 3.f * (2.f * zz - xx - yy) +
                                        SH_C3[4] * SHC(13, ch) * 4.f * 2.f * xz + SH_C3[5] * SHC(14, ch) * (xx - yy));
                        }
                    }
                }
            }
#undef SHC
#undef WR
            const float ddir[3] = {dx_[0] * dRGB[0] + dx_[1] * dRGB[1] + dx_[2] * dRGB[2],
                                   dy_[0] * dRGB[0] + dy_[1] * dRGB[1] + dy_[2] * dRGB[2],
                                   dz_[0] * dRGB[0] + dz_[1] * dRGB[1] + dz_[2] * dRGB[2]};
            float dm[3];
            dnormvdv3(dir_orig, ddir, dm);
            g[0] += dm[0]; g[1] += dm[1]; g[2] += dm[2];
        }
        dL_dmean3D[3 * idx] = g[0];
        dL_dmean3D[3 * idx + 1] = g[1];
        dL_dmean3D[3 * idx + 2] = g[2];
        if (scales) {
            const float* q = rotations + 4 * idx;
            const float r = q[0], x = q[1], y = q[2], z = q[3];
            const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                                   {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                                   {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
            const float s[3] = {scale_modifier * scales[3 * idx], scale_modifier * scales[3 * idx + 1],
                                scale_modifier * scales[3 * idx + 2]};
            float Mm[3][3], dM[3][3], dMt[3][3];
            for (int cc = 0; cc < 3; cc++) for (int rr = 0; rr < 3; rr++) Mm[cc][rr] = s[rr] * R[cc][rr];
            const float S[3][3] = {{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]},
                                   {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]},
                                   {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}};
            for (int cc = 0; cc < 3; cc++) for (int rr = 0; rr < 3; rr++)
                dM[cc][rr] = 2.0f * (Mm[0][rr] * S[cc][0] + Mm[1][rr] * S[cc][1] + Mm[2][rr] * S[cc][2]);
            for (int cc = 0; cc < 3; cc++) for (int rr = 0; rr < 3; rr++) dMt[cc][rr] = dM[rr][cc];
            for (int k = 0; k < 3; k++)
                dL_dscale[3 * idx + k] = R[0][k] * dMt[k][0] + R[1][k] * dMt[k][1] + R[2][k] * dMt[k][2];
            for (int k = 0; k < 3; k++) for (int rr = 0; rr < 3; rr++) dMt[k][rr] *= s[k];
            float* dq = dL_drot + 4 * idx;
            dq[0] = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
            dq[1] = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) - 4 * x * (dMt[2][2] + dMt[1][1]);
            dq[2] = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) - 4 * y * (dMt[2][2] + dMt[0][0]);
            dq[3] = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) - 4 * z * (dMt[1][1] + dMt[0][0]);
        }
    }
}

/* rasterizer_impl.cu:54-66 checkFrustum */
void oracle_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present) {
    for (int i = 0; i < P; i++)
        present[i] = xform_row(viewmatrix, 2, means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]) > 0.2f;
}

void oracle_set_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n > 0 ? n : 1);
#else
    (void)n;
#endif
}
int oracle_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
