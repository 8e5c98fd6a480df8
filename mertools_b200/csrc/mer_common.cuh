// mer_common.cuh — sm_90a building blocks shared by every kernel in libmer_b200.so.
//
// Thin inline-PTX wrappers (mbarrier, TMA, wgmma) plus the error plumbing of the
// C ABI declared in include/mer_b200.h.  Nothing here has a CPU fallback: every entry point
// of the library runs on the device or fails with a non-zero status.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

// --------------------------------------------------------------------------------------------
// host-side error plumbing
// --------------------------------------------------------------------------------------------
void mer_set_error(const char* fmt, ...);

#define MER_CUDA_CHECK(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      mer_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return 1;                                                                           \
    }                                                                                     \
  } while (0)

#define MER_REQUIRE(cond, ...)      \
  do {                              \
    if (!(cond)) {                  \
      mer_set_error(__VA_ARGS__);   \
      return 2;                     \
    }                               \
  } while (0)

// Build a tiled TMA descriptor (driver entry point resolved at run time; no -lcuda link dep).
// dims/strides are innermost-first; strides_bytes has rank-1 entries (dim 0 is contiguous).
int mer_make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int rank, const void* base,
                  const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                  CUtensorMapSwizzle swizzle);

int mer_num_sms();
void mer_count_launches(int n);  // cumulative count of kernels launched by this library

// --------------------------------------------------------------------------------------------
// device-side helpers
// --------------------------------------------------------------------------------------------
#ifdef __CUDACC__

#ifndef MER_SPIN_LIMIT
#define MER_SPIN_LIMIT (1u << 27)  // bounded mbarrier spin: trap instead of hanging the box
#endif

namespace mer {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe (try_wait may suspend the thread for a system-dependent time: wrong tool for a warp that polls
// several barriers and must react to whichever completes first)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > MER_SPIN_LIMIT) {
      printf("mer: mbarrier wait timed out (block %d thread %d)\n", (int)blockIdx.x,
             (int)threadIdx.x);
      __trap();
    }
  }
}
// same bound without the printf: a function call between wgmma instructions makes ptxas serialise them
__device__ __forceinline__ void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > MER_SPIN_LIMIT) __trap();
  }
}

// ---- TMA -----------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA; operands in shared memory, fp32 accumulators in registers) ----------
// Shared-memory matrix descriptor of a K-major operand tile laid out by TMA with SWIZZLE_128B: rows of 128 bytes,
// 8-row groups 1024 bytes apart (SBO), LBO unused (1).  bits: [0,14) addr>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 |
// [62,64) layout (1 = 128B swizzle).  Advancing the start address by 32 bytes steps K inside the swizzle row.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4) | (1ull << 16) | (uint64_t(1024 >> 4) << 32) |
         (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
__device__ __forceinline__ void wgmma_fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

#define MER_WGMMA_D64                                                                                            \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "  \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define MER_WGMMA_OUT64(d)                                                                                        \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),      \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),       \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),      \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),      \
      "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),      \
      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),      \
      "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),      \
      "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// D[64 x 128] (+)= A[64 x K-step] * B[128 x K-step]^T, both K-major in shared memory; one warpgroup issues.
// kind: 0 = f16 (k16), 1 = bf16 (k16), 2 = tf32 (k8).  accumulate = 0 overwrites D.
template <int KIND>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, int accumulate) {
  if (KIND == 0) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " MER_WGMMA_D64 ", %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : MER_WGMMA_OUT64(d)
                 : "l"(desc_a), "l"(desc_b), "r"(accumulate));
  } else if (KIND == 1) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " MER_WGMMA_D64 ", %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : MER_WGMMA_OUT64(d)
                 : "l"(desc_a), "l"(desc_b), "r"(accumulate));
  } else {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " MER_WGMMA_D64 ", %64, %65, p, 1, 1;\n}\n"
                 : MER_WGMMA_OUT64(d)
                 : "l"(desc_a), "l"(desc_b), "r"(accumulate));
  }
}

// ---- thread-block clusters ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- numerics ------------------------------------------------------------------------------
// round-to-nearest fp32 -> tf32 (result kept in an fp32 container; low 13 bits zero)
__device__ __forceinline__ float round_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
// two fp32 -> packed IEEE fp16 pair (round-to-nearest-even, saturating to +-65504): `lo` lands in the
// low half-word (the lower address)
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// fp32 -> (hi, lo) bf16 pair with x = hi + lo to 2^-17 relative: operand format of MER_GEMM_BF16X3.
// A split row of K values occupies the bytes of K fp32 values, organised in 128-byte groups of
// 32 values: [32 x bf16 hi | 32 x bf16 lo].  One 128B-swizzled TMA row therefore carries both halves
// of a 32-wide K block, exactly like a row of 32 fp32 values in TF32 mode.
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {  // low half <- a, high <- b
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ float bf16_round(float x) {
  return __uint_as_float(pack_bf16x2(x, 0.f) << 16);
}
// index (in bf16 units) of the hi half of logical column `col`; the lo half sits 32 further
__device__ __forceinline__ int split_index(int col) { return ((col >> 5) << 6) + (col & 31); }
// store 4 consecutive logical columns (col % 4 == 0) of a split row
__device__ __forceinline__ void store_split4(void* row_base, int col, float4 v) {
  const float hx = bf16_round(v.x), hy = bf16_round(v.y), hz = bf16_round(v.z), hw = bf16_round(v.w);
  uint16_t* o = reinterpret_cast<uint16_t*>(row_base) + split_index(col);
  *reinterpret_cast<uint2*>(o) = make_uint2(pack_bf16x2(hx, hy), pack_bf16x2(hz, hw));
  *reinterpret_cast<uint2*>(o + 32) =
      make_uint2(pack_bf16x2(v.x - hx, v.y - hy), pack_bf16x2(v.z - hz, v.w - hw));
}
__device__ __forceinline__ void store_split2(void* row_base, int col, float a, float b) {  // col % 2 == 0
  const uint32_t hp = pack_bf16x2(a, b);  // both hi halves in one conversion; as floats: the two 16-bit fields
  const float ha = __uint_as_float(hp << 16), hb = __uint_as_float(hp & 0xffff0000u);
  uint16_t* o = reinterpret_cast<uint16_t*>(row_base) + split_index(col);
  *reinterpret_cast<uint32_t*>(o) = hp;
  *reinterpret_cast<uint32_t*>(o + 32) = pack_bf16x2(a - ha, b - hb);
}
__device__ __forceinline__ void store_split1(void* row_base, int col, float v) {
  const float h = bf16_round(v);
  uint16_t* o = reinterpret_cast<uint16_t*>(row_base) + split_index(col);
  o[0] = (uint16_t)(__float_as_uint(h) >> 16);
  o[32] = (uint16_t)(pack_bf16x2(v - h, 0.f) & 0xFFFFu);
}

// exact (erf) GELU, as torch.nn.functional.gelu default
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
// erf-GELU for the GEMM epilogues, where the libdevice erff (~30 instructions, two branches) made the
// FC1 epilogue as long as its mainloop: Abramowitz-Stegun 7.1.26 (|erf error| <= 1.5e-7 in exact
// arithmetic); measured in fp32 over [-12, 12]: |gelu error| <= 4.7e-7 absolute, <= 2.9e-7 * |x| —
// three orders of magnitude below the TF32 / split-bf16 operand rounding that follows.
// One MUFU.RCP, one MUFU.EX2, 8 FMA-class ops.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * z * z));
  const float erf_abs = fmaf(-p * t, e, 1.0f);  // erf(|x| / sqrt 2)
  const float hx = 0.5f * x;
  return fmaf(fabsf(hx), erf_abs, hx);           // x/2 * (1 + sign(x) erf(|x|/sqrt 2))
}

// CLIP's quick_gelu: x * sigmoid(1.702 x), with ex2.approx / rcp.approx (|rel err| ~2e-7)
__device__ __forceinline__ float quick_gelu_fast(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.702f * 1.4426950408889634f * x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}

// ---- fp32 pairs (two lanes' worth of math on a 64-bit register pair, as the softmax / GELU code is written;
//      sm_90 has no paired fp32 instructions, so each pair op is two scalar ones) and the three-input max ----
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
__device__ __forceinline__ uint64_t pack2(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t add2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
// 2^x for two values on the FMA / ALU pipes instead of MUFU.EX2 (softmax kernels, where the 16 lanes of the XU
// pipe are the floor): x = n + f with n = round(x) taken from the mantissa of x + 1.5 * 2^23, f in [-0.5, 0.5],
// 2^f by a degree-4 polynomial (max relative error 2.7e-6 in fp32, below the fp16 / TF32 rounding of P that
// follows), 2^n added into the exponent field.  x is clamped to >= -126 (the result then rounds to 0 in P).
__device__ __forceinline__ void ex2_poly2(uint64_t x2, float& a, float& b) {
  float x0, x1;
  unpack2(x2, x0, x1);
  const uint64_t x = pack2(fmaxf(x0, -126.f), fmaxf(x1, -126.f));
  const auto bc = [](float v) { return pack2(v, v); };
  const uint64_t r = add2(x, bc(12582912.f));
  const uint64_t f = fma2(add2(r, bc(-12582912.f)), bc(-1.f), x);
  uint64_t p = fma2(bc(0.00957401655614376f), f, bc(0.055918190628290176f));
  p = fma2(p, f, bc(0.2402464896440506f));
  p = fma2(p, f, bc(0.6931217312812805f));
  p = fma2(p, f, bc(0.9999992847442627f));
  float p0, p1, r0, r1;
  unpack2(p, p0, p1);
  unpack2(r, r0, r1);
  a = __uint_as_float(__float_as_uint(p0) + (__float_as_uint(r0) << 23));
  b = __uint_as_float(__float_as_uint(p1) + (__float_as_uint(r1) << 23));
}
// gelu_erf_fast on two values at once.  Same polynomial; the constants of the first two steps are folded
// (0.3275911 / sqrt 2 and -log2(e) / 2), which moves individual results by at most an ulp of the intermediate.
__device__ __forceinline__ void gelu_erf_fast2(float x0, float x1, float& g0, float& g1) {
  const uint64_t x = pack2(x0, x1), ax = pack2(fabsf(x0), fabsf(x1));
  const auto bc = [](float v) { return pack2(v, v); };
  float d0, d1, t0, t1, a0, a1, e0, e1;
  unpack2(fma2(bc(0.3275911f * 0.70710678118654752440f), ax, bc(1.0f)), d0, d1);
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(d0));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(d1));
  const uint64_t t = pack2(t0, t1);
  uint64_t p = fma2(bc(-1.061405429f), t, bc(1.453152027f));  // -(a5 t + a4): the sign of erfc's series folded in
  p = fma2(p, t, bc(-1.421413741f));
  p = fma2(p, t, bc(0.284496736f));
  p = fma2(p, t, bc(-0.254829592f));
  unpack2(mul2(mul2(x, x), bc(-0.5f * 1.4426950408889634f)), a0, a1);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(a0));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(a1));
  const uint64_t erf_abs = fma2(mul2(p, t), pack2(e0, e1), bc(1.0f));  // erf(|x| / sqrt 2)
  unpack2(fma2(mul2(ax, bc(0.5f)), erf_abs, mul2(x, bc(0.5f))), g0, g1);
}

// torch.optim.Adam (coupled L2) on one parameter, in torch's operation order (lerp for the first moment, mul +
// addcmul for the second).  Every rounding step is explicit so that the fused and the stand-alone Adam kernels, compiled
// in different contexts, contract nothing differently and agree bit for bit.  bc1 = 1 - beta1^t,
// bc2_sqrt = sqrt(1 - beta2^t).  Returns the new parameter; m / v are updated in place.
__device__ __forceinline__ float adam_param(float pi, float grad, float& m, float& v, float lr, float beta1, float beta2,
                                            float eps, float wd, float bc1, float bc2_sqrt) {
  grad = __fmaf_rn(wd, pi, grad);
  m = __fmaf_rn(__fsub_rn(grad, m), __fsub_rn(1.f, beta1), m);
  v = __fmaf_rn(v, beta2, __fmul_rn(__fmul_rn(__fsub_rn(1.f, beta2), grad), grad));
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
  return __fsub_rn(pi, __fmul_rn(__fdiv_rn(lr, bc1), __fdiv_rn(m, denom)));
}

// The fusion nets' dropout keep-mask: element i of mask tensor m at step counter `step`, 1 (keep) with probability
// 1 - p.  A splitmix64 counter hash, the draw of fusion.cu:fus_dropout_mask_kernel with the tensor's 0x1000 (m + 1)
// folded into the seed; used by fusion_fused.cu and fusion_mlp.cu.
__device__ __forceinline__ float keep_hash(unsigned long long seed, int m, int step, long long i, float p) {
  unsigned long long z = seed + 0x1000ull * (unsigned long long)(m + 1) +
                         0x9E3779B97F4A7C15ull * (unsigned long long)(step + 1) +
                         0xD1B54A32D192ED03ull * (unsigned long long)(i + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  const float u = (float)(z >> 40) * (1.0f / 16777216.0f);
  return u >= p ? 1.f : 0.f;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace mer
#endif  // __CUDACC__
