// attention.cu — softmax(Q K^T / sqrt(64)) V for packed variable-length sequences, head_dim 64.
//
// Replaces HF eager/sdpa self-attention inside ViTLayer / HubertEncoderLayer / BertLayer
// (HF modeling_vit.py:171-196, modeling_hubert.py:262-345) as reached from the reference
// extractors (extract_vision_huggingface.py:143, extract_audio_huggingface.py:97,
// extract_text_huggingface.py:225).  No attention mask exists on this path: the reference feeds
// un-padded single sequences (audio/text) or equal-length frame batches (visual).
//
// Flash-style: one CTA = (sequence, head, 64-query block), 4 warps x 16 query rows; K/V blocks
// of 64 keys are double-buffered in shared memory with cp.async; S = QK^T and O += P V run on
// mma.sync.m16n8k8 TF32 with fp32 accumulation, online softmax in fp32 registers.  The S
// accumulator fragment is re-used directly as the A fragment of P V by permuting the key order
// inside each 8-key group (keys 2t / 2t+1 <-> k-columns t / t+4), with V rows fetched under the
// same permutation, so no shuffles or smem round-trip are needed.
// Used when the QKV GEMM wrote V into qkv (no V^T): CLIP L/14 rows in the fp16 stacks, MER_ATTENTION_LEGACY.
#include <stdlib.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int BQ = 64;
constexpr int BKV = 64;
constexpr int HD = 64;
constexpr int LDS = 68;  // padded row pitch (floats): conflict-free K and V fragment loads
constexpr int ATT_THREADS = 128;
constexpr int ATT_SMEM = 2 * 2 * BKV * LDS * 4;

__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem),
               "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

__global__ void __launch_bounds__(ATT_THREADS, 3)
attention_kernel(const float* __restrict__ qkv, float* __restrict__ ctx,
                 const int* __restrict__ cu_seqlens, int heads, int out_mode) {
  extern __shared__ __align__(16) float smem_f[];
  float* Ks = smem_f;                  // [2][BKV][LDS]
  float* Vs = smem_f + 2 * BKV * LDS;  // [2][BKV][LDS]

  const int seq = blockIdx.z;
  const int h = blockIdx.y;
  const int start = cu_seqlens[seq];
  const int len = cu_seqlens[seq + 1] - start;
  const int q0 = blockIdx.x * BQ;
  if (q0 >= len) return;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int g = lane >> 2;
  const int t = lane & 3;
  const int ld = 3 * heads * HD;
  const float* qbase = qkv + (long long)start * ld + h * HD;
  const float* kbase = qbase + heads * HD;
  const float* vbase = qbase + 2 * heads * HD;

  // ---- Q fragments (pre-scaled by 1/8: exact in tf32) ----
  uint32_t qa[8][4];
  {
    const int r_lo = min(q0 + warp * 16 + g, len - 1);
    const int r_hi = min(q0 + warp * 16 + g + 8, len - 1);
    const float* q_lo = qbase + (long long)r_lo * ld;
    const float* q_hi = qbase + (long long)r_hi * ld;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      qa[ks][0] = __float_as_uint(q_lo[ks * 8 + t] * 0.125f);
      qa[ks][1] = __float_as_uint(q_hi[ks * 8 + t] * 0.125f);
      qa[ks][2] = __float_as_uint(q_lo[ks * 8 + t + 4] * 0.125f);
      qa[ks][3] = __float_as_uint(q_hi[ks * 8 + t + 4] * 0.125f);
    }
  }

  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;

  const int n_kv = (len + BKV - 1) / BKV;

  auto load_tile = [&](int j, int buf) {
    const int kv0 = j * BKV;
    float* kd = Ks + buf * BKV * LDS;
    float* vd = Vs + buf * BKV * LDS;
#pragma unroll
    for (int i = 0; i < (BKV * HD / 4) / ATT_THREADS; ++i) {
      const int idx = tid + i * ATT_THREADS;  // float4 index inside the 64x64 tile
      const int r = idx >> 4;
      const int c4 = idx & 15;
      const int key = kv0 + r;
      const int ok = key < len ? 16 : 0;
      const long long goff = (long long)min(key, len - 1) * ld + c4 * 4;
      cp_async16(kd + r * LDS + c4 * 4, kbase + goff, ok);
      cp_async16(vd + r * LDS + c4 * 4, vbase + goff, ok);
    }
    cp_async_commit();
  };

  load_tile(0, 0);
  constexpr float LOG2E = 1.4426950408889634f;

  for (int j = 0; j < n_kv; ++j) {
    const int buf = j & 1;
    if (j + 1 < n_kv) {
      load_tile(j + 1, buf ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* kt = Ks + buf * BKV * LDS;
    const float* vt = Vs + buf * BKV * LDS;

    // ---- S = (Q/8) K^T : 16 x 64 per warp ----
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      const float* kr = kt + (nt * 8 + g) * LDS + t;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        mma_tf32(s[nt], qa[ks], __float_as_uint(kr[ks * 8]), __float_as_uint(kr[ks * 8 + 4]));
      }
    }
    // ---- mask the tail block ----
    const int kv0 = j * BKV;
    if (kv0 + BKV > len) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int key = kv0 + nt * 8 + 2 * t;
        if (key >= len) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
        if (key + 1 >= len) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      }
    }
    // ---- online softmax ----
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx_lo = fmaxf(mx_lo, fmaxf(s[nt][0], s[nt][1]));
      mx_hi = fmaxf(mx_hi, fmaxf(s[nt][2], s[nt][3]));
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
    const float mn_lo = fmaxf(m_lo, mx_lo);
    const float mn_hi = fmaxf(m_hi, mx_hi);
    const float sc_lo = exp2f((m_lo - mn_lo) * LOG2E);
    const float sc_hi = exp2f((m_hi - mn_hi) * LOG2E);
    m_lo = mn_lo;
    m_hi = mn_hi;
    float ps_lo = 0.f, ps_hi = 0.f;
    const float ml2_lo = mn_lo * LOG2E, ml2_hi = mn_hi * LOG2E;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = exp2f(fmaf(s[nt][0], LOG2E, -ml2_lo));
      s[nt][1] = exp2f(fmaf(s[nt][1], LOG2E, -ml2_lo));
      s[nt][2] = exp2f(fmaf(s[nt][2], LOG2E, -ml2_hi));
      s[nt][3] = exp2f(fmaf(s[nt][3], LOG2E, -ml2_hi));
      ps_lo += s[nt][0] + s[nt][1];
      ps_hi += s[nt][2] + s[nt][3];
    }
    l_lo = l_lo * sc_lo + ps_lo;
    l_hi = l_hi * sc_hi + ps_hi;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      o[dt][0] *= sc_lo; o[dt][1] *= sc_lo; o[dt][2] *= sc_hi; o[dt][3] *= sc_hi;
    }
    // ---- O += P V (keys permuted inside each group of 8: col t <-> key 2t, col t+4 <-> key 2t+1) ----
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      uint32_t pa[4];
      pa[0] = __float_as_uint(round_tf32(s[ks][0]));
      pa[1] = __float_as_uint(round_tf32(s[ks][2]));
      pa[2] = __float_as_uint(round_tf32(s[ks][1]));
      pa[3] = __float_as_uint(round_tf32(s[ks][3]));
      const float* vr0 = vt + (ks * 8 + 2 * t) * LDS + g;
      const float* vr1 = vr0 + LDS;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) {
        mma_tf32(o[dt], pa, __float_as_uint(vr0[dt * 8]), __float_as_uint(vr1[dt * 8]));
      }
    }
    __syncthreads();  // everyone done with buf before the next prefetch overwrites it
  }

  // ---- finalize ----
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
  const float inv_lo = 1.0f / l_lo;
  const float inv_hi = 1.0f / l_hi;
  const int row_lo = q0 + warp * 16 + g;
  const int row_hi = row_lo + 8;
  const int ldc = heads * HD;
  float* c_lo = ctx + (long long)(start + row_lo) * ldc + h * HD + 2 * t;
  float* c_hi = ctx + (long long)(start + row_hi) * ldc + h * HD + 2 * t;
#pragma unroll
  for (int dt = 0; dt < 8; ++dt) {
    float2 a = make_float2(o[dt][0] * inv_lo, o[dt][1] * inv_lo);
    float2 b = make_float2(o[dt][2] * inv_hi, o[dt][3] * inv_hi);
    if (out_mode == 2) {  // split bf16 rows for a BF16X3 out-proj GEMM
      const int col = h * HD + dt * 8 + 2 * t;
      if (row_lo < len) store_split2(ctx + (long long)(start + row_lo) * ldc, col, a.x, a.y);
      if (row_hi < len) store_split2(ctx + (long long)(start + row_hi) * ldc, col, b.x, b.y);
      continue;
    }
    if (out_mode == 1) {
      a.x = round_tf32(a.x); a.y = round_tf32(a.y); b.x = round_tf32(b.x); b.y = round_tf32(b.y);
    }
    if (row_lo < len) *reinterpret_cast<float2*>(c_lo + dt * 8) = a;
    if (row_hi < len) *reinterpret_cast<float2*>(c_hi + dt * 8) = b;
  }
}

}  // namespace

bool mer_attention_legacy() {
  static const bool legacy = getenv("MER_ATTENTION_LEGACY") != nullptr;
  return legacy;
}

bool mer_attention_uses_tc(int max_seqlen) {
  return !mer_attention_legacy() && max_seqlen <= 253;
}

int mer_attention_launch(const float* qkv, const float* vt, long long vt_ld, float* ctx,
                         const int* cu_seqlens, int n_seq, long long tokens, int max_seqlen, int heads,
                         int flags, cudaStream_t stream) {
  MER_REQUIRE(qkv && ctx && cu_seqlens, "mer_attention: null operand");
  const int out_mode = (flags & MER_EPI_OUT_F16) ? 3 : (flags & MER_EPI_SPLIT_BF16) ? 2 : ((flags & MER_EPI_ROUND_TF32) ? 1 : 0);
  if (flags & MER_ATT_QKV_F16) {
    // fp16 q | k rows and V^T (attention_f16.cu), ctx in any operand format: the fp16 stacks, and the TF32 / BF16X3
    // stacks for rows of 254 .. 505 tokens
    MER_REQUIRE(vt && mer_attention_f16_supported(max_seqlen),
                "mer_attention: fp16 inputs need V^T and sequences <= 505 tokens (max_seqlen %d)", max_seqlen);
    return mer_attention_f16_launch(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode, stream);
  }
  // sequences of up to 253 tokens (ViT 197, HuBERT 5 s = 249, most sentences) with V^T written by the QKV GEMM
  // (which then leaves the V columns of qkv unwritten): the tf32 form of the V^T kernel
  if (vt && mer_attention_uses_tc(max_seqlen))
    return mer_attention_tc_launch(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode, stream);
  MER_REQUIRE(!(flags & MER_EPI_OUT_F16),
              "mer_attention: fp16 ctx needs V^T (sequences <= 253 tokens)");
  MER_REQUIRE(heads > 0 && heads <= 65535 && n_seq <= 65535, "mer_attention: bad grid (%d heads, %d seqs)",
              heads, n_seq);
  if (n_seq <= 0 || max_seqlen <= 0) return 0;
  static MerPerDevice attr_set;
  if (attr_set.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        ATT_SMEM));
    attr_set.mark();
  }
  dim3 grid((max_seqlen + BQ - 1) / BQ, heads, n_seq);
  attention_kernel<<<grid, ATT_THREADS, ATT_SMEM, stream>>>(qkv, ctx, cu_seqlens, heads,
                                                           (flags & MER_EPI_SPLIT_BF16) ? 2 : ((flags & MER_EPI_ROUND_TF32) ? 1 : 0));
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}
