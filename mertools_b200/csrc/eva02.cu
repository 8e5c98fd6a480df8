// eva02.cu — the two kernels of timm's EVA02 blocks (eva02_base_patch14_224, the visual extractor's EVACLIP_VIT) that
// the shared stack does not have: the 2D rotary embedding with interleaved pairs on the fp16 q | k columns of the QKV
// GEMM output, and the SwiGLU gate followed by the LayerNorm over the gated product (timm SwiGLU with norm_layer).
// Both run inside mer_run_stack when MerStackArgs carries a rope table / FFN norms (the MER_VISION_EVA02 tower).
#include <cuda_fp16.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int ROPE_THREADS = 128;

// timm apply_rot_embed_cat on one token: for every q and k head and pair i < 32,
// (x[2i], x[2i+1]) -> (x[2i] c - x[2i+1] s, x[2i+1] c + x[2i] s), c / s = cos_t / sin_t[patch, i].  Tokens are packed
// frames of tpf rows; the first `prefix` rows of a frame (the class row) are left alone.  One CTA per token, each thread
// two adjacent pairs (one 8-byte word), fp32 math rounded once to fp16.
__global__ void __launch_bounds__(ROPE_THREADS)
rope2d_kernel(uint16_t* __restrict__ qkv, long long ld, int tpf, int prefix, int heads, const float* __restrict__ cos_t,
              const float* __restrict__ sin_t) {
  const long long tok = blockIdx.x;
  const int p = (int)(tok % tpf) - prefix;
  if (p < 0) return;
  uint16_t* row = qkv + tok * ld;
  const float4* cr = reinterpret_cast<const float4*>(cos_t + (long long)p * 32);
  const float4* sr = reinterpret_cast<const float4*>(sin_t + (long long)p * 32);
  const int words = 2 * heads * 16;  // q and k heads x 16 words of two pairs
  for (int u = threadIdx.x; u < words; u += ROPE_THREADS) {
    const int hh = u >> 4, w = u & 15;  // head, word inside the head (pairs 2w, 2w + 1)
    uint2* a = reinterpret_cast<uint2*>(row + hh * 64 + 4 * w);
    const uint2 v = *a;
    const float2 x01 = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
    const float2 x23 = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
    const float4 c4 = __ldg(cr + (w >> 1)), s4 = __ldg(sr + (w >> 1));
    const float c0 = (w & 1) ? c4.z : c4.x, c1 = (w & 1) ? c4.w : c4.y;
    const float s0 = (w & 1) ? s4.z : s4.x, s1 = (w & 1) ? s4.w : s4.y;
    *a = make_uint2(pack_f16x2(x01.x * c0 - x01.y * s0, x01.y * c0 + x01.x * s0),
                    pack_f16x2(x23.x * c1 - x23.y * s1, x23.y * c1 + x23.x * s1));
  }
}

constexpr int SGLN_THREADS = 256;
constexpr int SGLN_MAX = 4096;                               // widest gated product
constexpr int SGLN_VEC = SGLN_MAX / 4 / SGLN_THREADS;       // float4 of the product per thread at that width

__device__ __forceinline__ float sgln_block_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < SGLN_THREADS / 32; ++i) t += red[i];
  return t;
}

__device__ __forceinline__ float silu_mul(float g, float x) { return g / (1.0f + expf(-g)) * x; }

// y = LayerNorm(silu(in[:, :H]) * in[:, H:]) * gamma + beta, one CTA per row: the product stays in registers between
// the mean, the centred variance (both fp32) and the write.  Output fp16 (OUT_F16) or tf32-rounded fp32.
template <bool OUT_F16>
__global__ void __launch_bounds__(SGLN_THREADS)
swiglu_ln_kernel(const float* __restrict__ in, const float* __restrict__ gamma, const float* __restrict__ beta,
                 float eps, void* __restrict__ out, int H) {
  __shared__ float red[2][SGLN_THREADS / 32];
  const long long row = blockIdx.x;
  const int n4 = H >> 2, tid = threadIdx.x;
  const float4* g4 = reinterpret_cast<const float4*>(in + row * 2 * H);
  const float4* x4 = g4 + n4;
  float4 v[SGLN_VEC];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < SGLN_VEC; ++i) {
    const int c = tid + i * SGLN_THREADS;
    if (c < n4) {
      const float4 g = __ldcs(g4 + c), x = __ldcs(x4 + c);
      v[i] = make_float4(silu_mul(g.x, x.x), silu_mul(g.y, x.y), silu_mul(g.z, x.z), silu_mul(g.w, x.w));
    } else {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = sgln_block_sum(s, red[0]) / (float)H;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < SGLN_VEC; ++i) {
    if (tid + i * SGLN_THREADS < n4) {
      v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
      ss = fmaf(v[i].x, v[i].x, ss);
      ss = fmaf(v[i].y, v[i].y, ss);
      ss = fmaf(v[i].z, v[i].z, ss);
      ss = fmaf(v[i].w, v[i].w, ss);
    }
  }
  const float r = rsqrtf(sgln_block_sum(ss, red[1]) / (float)H + eps);
  const float4* ga = reinterpret_cast<const float4*>(gamma);
  const float4* be = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < SGLN_VEC; ++i) {
    const int c = tid + i * SGLN_THREADS;
    if (c >= n4) continue;
    const float4 g = __ldg(ga + c), b = __ldg(be + c);
    const float4 o = make_float4(fmaf(v[i].x * r, g.x, b.x), fmaf(v[i].y * r, g.y, b.y), fmaf(v[i].z * r, g.z, b.z),
                                 fmaf(v[i].w * r, g.w, b.w));
    if (OUT_F16)
      reinterpret_cast<uint2*>(out)[row * n4 + c] = make_uint2(pack_f16x2(o.x, o.y), pack_f16x2(o.z, o.w));
    else
      reinterpret_cast<float4*>(out)[row * n4 + c] =
          make_float4(round_tf32(o.x), round_tf32(o.y), round_tf32(o.z), round_tf32(o.w));
  }
}

// begins[i] = i * step + skip, ends[i] = (i + 1) * step: the rows of each packed frame after its first `skip`
__global__ void frame_spans_kernel(int* begins, int* ends, int n, int step, int skip) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    begins[i] = i * step + skip;
    ends[i] = (i + 1) * step;
  }
}

}  // namespace

int mer_frame_spans_launch(int* begins, int* ends, int n, int step, int skip, cudaStream_t stream) {
  frame_spans_kernel<<<(n + 255) / 256, 256, 0, stream>>>(begins, ends, n, step, skip);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_rope2d_f16(void* qkv16, long long ld, long long tokens, int tokens_per_frame, int prefix, int heads,
                              int head_dim, const float* cos_t, const float* sin_t, int table_rows, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(qkv16 && cos_t && sin_t, "mer_rope2d_f16: null operand");
  MER_REQUIRE(head_dim == 64, "mer_rope2d_f16: head_dim %d (64 only)", head_dim);
  MER_REQUIRE(heads > 0 && ld >= 2ll * heads * 64 && ld % 4 == 0 && (reinterpret_cast<uintptr_t>(qkv16) & 7) == 0,
              "mer_rope2d_f16: bad row layout (%d heads, ld %lld)", heads, ld);
  MER_REQUIRE(tokens_per_frame > 0 && prefix >= 0 && tokens > 0 && tokens < (1ll << 31) && tokens % tokens_per_frame == 0,
              "mer_rope2d_f16: %lld tokens are not whole frames of %d", tokens, tokens_per_frame);
  MER_REQUIRE(table_rows == tokens_per_frame - prefix && (reinterpret_cast<uintptr_t>(cos_t) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(sin_t) & 15) == 0,
              "mer_rope2d_f16: table of %d rows for %d rotated rows per frame (16-byte aligned tables)", table_rows,
              tokens_per_frame - prefix);
  rope2d_kernel<<<(unsigned)tokens, ROPE_THREADS, 0, stream>>>(static_cast<uint16_t*>(qkv16), ld, tokens_per_frame,
                                                               prefix, heads, cos_t, sin_t);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_swiglu_ln(const float* in, const float* gamma, const float* beta, float eps, void* out,
                             long long rows, int hidden, int out_f16, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(in && gamma && beta && out, "mer_swiglu_ln: null operand");
  MER_REQUIRE(hidden > 0 && hidden % 128 == 0 && hidden <= SGLN_MAX, "mer_swiglu_ln: width %d (a multiple of 128 up to %d)",
              hidden, SGLN_MAX);
  MER_REQUIRE(rows > 0 && rows < (1ll << 31), "mer_swiglu_ln: %lld rows", rows);
  MER_REQUIRE(static_cast<const void*>(in) != out, "mer_swiglu_ln: out may not alias in");
  if (out_f16)
    swiglu_ln_kernel<true><<<(unsigned)rows, SGLN_THREADS, 0, stream>>>(in, gamma, beta, eps, out, hidden);
  else
    swiglu_ln_kernel<false><<<(unsigned)rows, SGLN_THREADS, 0, stream>>>(in, gamma, beta, eps, out, hidden);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}
