// TF32 tensor-core helpers shared by the 1x1 decoder (feature_decoder.cu) and the text query (feature_query.cu).
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

#include "common.cuh"

namespace f3dgs {

__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

// d += a * b, m16n8k8 TF32, fp32 accumulate.  Fragments (PTX ISA, mma.m16n8k8 .tf32), g = lane >> 2, t = lane & 3:
//   a0 (g, t)  a1 (g + 8, t)  a2 (g, t + 4)  a3 (g + 8, t + 4)      b0 (k = t, n = g)  b1 (k = t + 4, n = g)
//   d0 (g, 2t) d1 (g, 2t + 1) d2 (g + 8, 2t) d3 (g + 8, 2t + 1)
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// float16 data is upcast exactly where it is loaded, so a float16 input gives the result of its float32 upcast
__device__ __forceinline__ float load_f32(const float* p) { return __ldg(p); }
__device__ __forceinline__ float load_f32(const __half* p) { return __half2float(__ldg(p)); }

}  // namespace f3dgs
