// Shared device helpers for the f3dgs kernels (sm_90a).
//
// Numerics contract.  The tile/key indexing of this library must be bit-identical to the
// reference extension built by nvcc with default flags (-fmad=true, IEEE div/sqrt).  Where a*b+c
// becomes an FMA is decided twice: by NVVM (visible in PTX as fma.rn) and again by ptxas, which
// fuses un-suffixed mul.f32/add.f32 pairs it finds in the PTX.  Explicit _rn intrinsics would
// block the second step, so the bit-exact stages (forward preprocess, the alpha/T recurrence of
// the composite) are written as plain fp32 expressions with the same expression trees as the
// reference's formulas and compiled by the same compiler with the same flags; bit-identity of
// radii / keys / n_contrib / final_T / colour / depth against the reference build is then
// checked on the GPU (tests/test_gpu_parity.py).  The CPU oracle (oracle/f3dgs_oracle.c)
// restates the resulting operation sequence with fmaf().
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define F3DGS_TILE_X 16
#define F3DGS_TILE_Y 16

namespace f3dgs {

// ---------------------------------------------------------------- host launch arithmetic
// scratch buffers are carved into sub-buffers that start on 256-byte boundaries
inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }
// CTAs of 256 threads for one thread per work item
inline unsigned blocks_for(long long threads) { return (unsigned)((threads + 255) / 256); }

// ---------------------------------------------------------------- exact fp32 building blocks
__device__ __forceinline__ float mulr(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float addr(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float subr(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fmar(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float divr(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float rcpr(float a) { return __frcp_rn(a); }
__device__ __forceinline__ float sqrtr(float a) { return __fsqrt_rn(a); }
// Two independent fma.rn on a pair of accumulators.  The feature loops keep the two pixels of a quad row in one float2;
// each half is an IEEE fma.rn, so the result is bit-identical to two scalar fmaf calls.
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// a0*b0 + a1*b1 + a2*b2 as nvcc contracts it in the reference (GLM mat3 products, dot(),
// transformPoint): the middle product is a plain multiply, the other two are fused.
__device__ __forceinline__ float dot3r(float a0, float b0, float a1, float b1, float a2, float b2) {
    return fmar(a2, b2, fmar(a0, b0, mulr(a1, b1)));
}

// reference auxiliary.h:58-66 (transformPoint4x3), row `r` of the column-major 4x4
__device__ __forceinline__ float xform_row(const float* __restrict__ m, int r, float x, float y, float z) {
    return addr(m[12 + r], fmar(z, m[8 + r], fmar(x, m[r], mulr(y, m[4 + r]))));
}

// reference auxiliary.h:41-44 (ndc2Pix): evaluated in double because of the unsuffixed literals
__device__ __forceinline__ float ndc2pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

// reference auxiliary.h:46-56 (getRect): float divide by the int tile size, truncation, clamp
__device__ __forceinline__ void tile_rect(float px, float py, int max_radius, uint32_t gx, uint32_t gy,
                                          uint32_t& x0, uint32_t& y0, uint32_t& x1, uint32_t& y1) {
    x0 = min(gx, (uint32_t)max((int)0, (int)((px - max_radius) / F3DGS_TILE_X)));
    y0 = min(gy, (uint32_t)max((int)0, (int)((py - max_radius) / F3DGS_TILE_Y)));
    x1 = min(gx, (uint32_t)max((int)0, (int)((px + max_radius + F3DGS_TILE_X - 1) / F3DGS_TILE_X)));
    y1 = min(gy, (uint32_t)max((int)0, (int)((py + max_radius + F3DGS_TILE_Y - 1) / F3DGS_TILE_Y)));
}

// ---------------------------------------------------------------- mbarrier / bulk-copy PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(
                     smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
// try_wait with a suspend-time hint: the warp is parked by the hardware until the phase completes
// (or the hint expires) instead of spinning and stealing issue slots from the warps it waits for.
// The whole wait loop is one asm block: written as a C loop the compiler re-materialises the barrier address (S2R
// SR_CgaCtaId, LEA, ...) inside it, 17 instructions per poll, and waiting warps then take a quarter of the SM's issue
// slots from the warps they wait for (ncu source counters).  Here a poll is TRYWAIT + NANOSLEEP + BRA.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "F3DGS_WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@p bra F3DGS_DONE_%=;\n\t"
        "bra F3DGS_WAIT_%=;\n\t"
        "F3DGS_DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
        "r"(parity), "r"(0x989680u)
        : "memory");
}
// Wait with a real sleep between polls, for roles that are far ahead of / behind their partner (epilogue waiting for a whole
// tile, producer waiting for a free stage, ...).  The poll loop of mbar_wait costs three issue slots every ~20 cycles per
// waiting warp: with ten waiting warps per SM that was 43% of all instructions executed by a forward composite kernel
// (ncu source counters), taken from the warps on the critical path.  `ns` bounds the added wake-up latency.
__device__ __forceinline__ void mbar_wait_sleep(uint64_t* bar, uint32_t parity, uint32_t ns) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "F3DGS_SWAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra F3DGS_SDONE_%=;\n\t"
        "nanosleep.u32 %2;\n\t"
        "bra F3DGS_SWAIT_%=;\n\t"
        "F3DGS_SDONE_%=:\n\t}" ::"r"(smem_u32(bar)),
        "r"(parity), "r"(ns)
        : "memory");
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// ---------------------------------------------------------------- vector global access
__device__ __forceinline__ void st_na_f4(float* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}
// one full 32-byte sector per lane, as two 128-bit stores (the widest global store of sm_90); p 32-byte aligned
__device__ __forceinline__ void st_na_f8(float* p, float4 a, float4 b) {
    st_na_f4(p, a);
    st_na_f4(p + 4, b);
}
__device__ __forceinline__ float4 ld_nc_f4(const float* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ void red_add_f4(float* p, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void red_add_f1(float* p, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// Per-Gaussian record produced by the forward preprocess and consumed by both composites.
// 48 bytes, three 16-byte words so it can be moved with 128-bit accesses.
struct __align__(16) SplatRec {
    float x, y;        // pixel-space mean (reference geom.means2D)
    float ex, ey;      // conservative half extents of the region where alpha >= 1/255
    float ca, cb, cc;  // conic (reference geom.conic_opacity.xyz)
    float op;          // opacity (conic_opacity.w)
    float r, g, b;     // colour after SH eval/clamp, or colors_precomp
    float depth;       // view-space z (reference geom.depths)
};

}  // namespace f3dgs
