// attention_mma.cuh — warp-level mma.sync helpers shared by the relative-position attention kernels
// (attention_rel.cu, attention_xl.cu): fp16 m16n8k16 and tf32 m16n8k8 products, 16-byte cp.async, ex2.approx, and the
// A-fragment / 8-row product loaders for 64-wide head rows in shared or global memory.
#pragma once

#include <stdint.h>

#include "mer_common.cuh"

namespace mer {

__device__ __forceinline__ void mma_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// A fragments (16 rows x 64 head dims) of rows lo / hi (row-major, 64 contiguous elements each)
template <bool F16, typename T>
__device__ __forceinline__ void load_a(uint32_t (&a)[F16 ? 4 : 8][4], const T* lo, const T* hi, int t) {
#pragma unroll
  for (int ks = 0; ks < (F16 ? 4 : 8); ++ks) {
    if (F16) {
      const uint32_t* l = reinterpret_cast<const uint32_t*>(lo + ks * 16);
      const uint32_t* h = reinterpret_cast<const uint32_t*>(hi + ks * 16);
      a[ks][0] = l[t]; a[ks][1] = h[t]; a[ks][2] = l[t + 4]; a[ks][3] = h[t + 4];
    } else {
      const uint32_t* l = reinterpret_cast<const uint32_t*>(lo) + ks * 8;
      const uint32_t* h = reinterpret_cast<const uint32_t*>(hi) + ks * 8;
      a[ks][0] = l[t]; a[ks][1] = h[t]; a[ks][2] = l[t + 4]; a[ks][3] = h[t + 4];
    }
  }
}

// c (16 x 8) = A (16 x 64) . B^T for the 8 rows of b starting at b (pitch LDS), then stored to out rows r / r + 8
template <bool F16, typename T, int LDS>
__device__ __forceinline__ void mma_row8(float (&c)[4], const uint32_t (&a)[F16 ? 4 : 8][4], const T* b, int g, int t) {
  c[0] = c[1] = c[2] = c[3] = 0.f;
  const T* br = b + g * LDS;
#pragma unroll
  for (int ks = 0; ks < (F16 ? 4 : 8); ++ks) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(br + ks * (F16 ? 16 : 8));
    if (F16)
      mma_f16(c, a[ks], w[t], w[t + 4]);
    else
      mma_tf32(c, a[ks], w[t], w[t + 4]);
  }
}

}  // namespace mer
