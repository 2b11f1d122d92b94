// Tensor-core helpers of the forward composite's feature contraction (composite_fwd.cu, TC feature warps).
//
// The feature contraction of a pixel block,  out[ch, px] = sum_k f[k, ch] * w[k, px]  over the block's instances, is a
// dense GEMM once the blend weights of the pairs that did not blend are written as zeros.  It runs on the tensor cores
// (warp-level mma.sync m16n8k8, TF32 inputs, fp32 accumulate) as an ERROR-COMPENSATED TF32 product: every fp32 operand
// x is split into hi = x with the 13 low mantissa bits cleared (exactly a TF32 number) and lo = x - hi (exact in fp32),
// and
//      a * b  ~=  a_hi * b_hi + a_hi * b_lo + a_lo * b_hi                    (three TF32 MMAs, fp32 accumulate)
// The dropped a_lo * b_lo term and the truncation of the lo parts to TF32 are each <= 2^-21 |a b|; the three products
// themselves are exact in fp32 (11 x 11 significant bits).  That is ~200x inside the 1e-4 relative parity bound.
#pragma once
#include <stdint.h>

#include "common.cuh"

namespace f3dgs {

// hi / lo split of an fp32 value for the compensated TF32 product
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// d (+)= a * b, m16n8k8, A row-major 16x8 (4 regs), B column-major 8x8 (2 regs), D 16x8 fp32 (4 regs).  Fragments
// (PTX ISA, mma.m16n8k8 .tf32), g = lane >> 2, t = lane & 3:
//   a0 (g, t)  a1 (g + 8, t)  a2 (g, t + 4)  a3 (g + 8, t + 4)      b0 (k = t, n = g)  b1 (k = t + 4, n = g)
//   d0 (g, 2t) d1 (g, 2t + 1) d2 (g + 8, 2t) d3 (g + 8, 2t + 1)
__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

}  // namespace f3dgs
