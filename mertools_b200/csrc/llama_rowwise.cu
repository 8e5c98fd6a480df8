// llama_rowwise.cu — the element- and row-wise kernels of a LLaMA decoder layer (HF modeling_llama.py) that the GEMM
// and the causal attention kernel do not cover: RMSNorm over wide fp32 residual rows, the rotate-half rotary embedding
// in place on the fp16 q | k columns of the QKV GEMM output, and the SwiGLU gate with an fp16 output.  Used by the
// LLaMA text extractor (mertools_b200/extract/llama_text.py, reference extract_text_huggingface.py:170-196).  Also the
// wide nn.LayerNorm (fp16 / fp32 / accumulate outputs) of the BLOOM / OPT decoders (extract/ln_decoder_text.py), and
// its form over the valid columns of padded rows and the head-dim-64 rotary embedding of Falcon's multi-query layout.
#include <cuda_fp16.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int RMS_THREADS = 256;
constexpr int RMS_MAX_DIM = 8192;
constexpr int RMS_VEC = RMS_MAX_DIM / 4 / RMS_THREADS;  // float4 per thread at the widest row

// LlamaRMSNorm: y = w * (x * rsqrt(mean(x^2) + eps)), mean(x^2) in fp32.  One CTA per row; the row stays in
// registers between the reduction and the write, so x is read from HBM once.
__global__ void __launch_bounds__(RMS_THREADS)
rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, uint16_t* __restrict__ y16,
               float* __restrict__ acc, int dim, float eps) {
  __shared__ float red[RMS_THREADS / 32];
  const long long row = blockIdx.x;
  const int n4 = dim >> 2, tid = threadIdx.x;
  const float4* xr = reinterpret_cast<const float4*>(x + row * dim);
  float4 v[RMS_VEC];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < RMS_VEC; ++i) {
    const int c = tid + i * RMS_THREADS;
    v[i] = c < n4 ? __ldcs(xr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    ss = fmaf(v[i].x, v[i].x, ss);
    ss = fmaf(v[i].y, v[i].y, ss);
    ss = fmaf(v[i].z, v[i].z, ss);
    ss = fmaf(v[i].w, v[i].w, ss);
  }
  ss = warp_sum(ss);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < RMS_THREADS / 32; ++i) tot += red[i];
  const float r = rsqrtf(tot / (float)dim + eps);
  const float4* w4 = reinterpret_cast<const float4*>(w);
#pragma unroll
  for (int i = 0; i < RMS_VEC; ++i) {
    const int c = tid + i * RMS_THREADS;
    if (c >= n4) break;
    const float4 g = __ldg(w4 + c);
    const float4 o = make_float4(g.x * (v[i].x * r), g.y * (v[i].y * r), g.z * (v[i].z * r), g.w * (v[i].w * r));
    if (y16) *reinterpret_cast<uint2*>(y16 + row * dim + 4 * c) = make_uint2(pack_f16x2(o.x, o.y), pack_f16x2(o.z, o.w));
    if (acc) {
      float4* a = reinterpret_cast<float4*>(acc + row * dim) + c;
      float4 s = *a;
      s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
      *a = s;
    }
  }
}

__device__ __forceinline__ float block_sum(float v, float* red) {  // red: RMS_THREADS / 32 floats, reusable after
  v = warp_sum(v);
  const int tid = threadIdx.x;
  if ((tid & 31) == 0) red[tid >> 5] = v;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < RMS_THREADS / 32; ++i) tot += red[i];
  return tot;
}

// nn.LayerNorm of the pre-LN decoders (BLOOM, OPT): y = (x - mean) * rsqrt(var + eps) * gamma + beta with the mean and
// the biased variance as two passes over the row held in registers (x is read from HBM once).  One CTA per row.
// PITCHED: x and every output are rows of pitch ld >= dim (Falcon's residual rows padded to a multiple of 128 columns);
// only the dim valid columns are read or written.  PITCHED = false is the kernel of mer_layernorm_f16, rows of pitch dim.
template <bool PITCHED>
__global__ void __launch_bounds__(RMS_THREADS)
layernorm_f16_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                     uint16_t* __restrict__ y16, float* __restrict__ y32, float* __restrict__ acc, int dim, float eps,
                     long long ld) {
  __shared__ float red[2][RMS_THREADS / 32];
  const long long row = PITCHED ? blockIdx.x * ld : (long long)blockIdx.x * dim;  // offset of the row (elements)
  const int n4 = dim >> 2, tid = threadIdx.x;
  const float4* xr = reinterpret_cast<const float4*>(x + row);
  float4 v[RMS_VEC];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < RMS_VEC; ++i) {
    const int c = tid + i * RMS_THREADS;
    v[i] = c < n4 ? __ldcs(xr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = block_sum(s, red[0]) / (float)dim;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < RMS_VEC; ++i) {
    const int c = tid + i * RMS_THREADS;
    if (c >= n4) break;
    v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
    ss = fmaf(v[i].x, v[i].x, ss);
    ss = fmaf(v[i].y, v[i].y, ss);
    ss = fmaf(v[i].z, v[i].z, ss);
    ss = fmaf(v[i].w, v[i].w, ss);
  }
  const float r = rsqrtf(block_sum(ss, red[1]) / (float)dim + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < RMS_VEC; ++i) {
    const int c = tid + i * RMS_THREADS;
    if (c >= n4) break;
    const float4 g = __ldg(g4 + c), b = __ldg(b4 + c);
    const float4 o = make_float4(fmaf(v[i].x * r, g.x, b.x), fmaf(v[i].y * r, g.y, b.y), fmaf(v[i].z * r, g.z, b.z),
                                 fmaf(v[i].w * r, g.w, b.w));
    if (y16) *reinterpret_cast<uint2*>(y16 + row + 4 * c) = make_uint2(pack_f16x2(o.x, o.y), pack_f16x2(o.z, o.w));
    if (y32) reinterpret_cast<float4*>(y32 + row)[c] = o;
    if (acc) {
      float4* a = reinterpret_cast<float4*>(acc + row) + c;
      float4 t = *a;
      t.x += o.x; t.y += o.y; t.z += o.z; t.w += o.w;
      *a = t;
    }
  }
}

__device__ __forceinline__ float2 f16x2_to_float2(uint32_t u) {
  return __half22float2(*reinterpret_cast<const __half2*>(&u));
}

// Rotate-half RoPE (HF apply_rotary_pos_emb) at head_dim HD: for j < HD / 2,
// (x_j, x_{j+HD/2}) -> (x_j c - x_{j+HD/2} s, x_{j+HD/2} c + x_j s) with c = cos_t[pos, j], s = sin_t[pos, j].  One CTA
// per token; each thread rotates two adjacent j of one head, in fp32, rounding once to fp16.  The heads rotated are the
// first 2 * heads of the row (QK: LLaMA's q and k blocks of `heads` heads each) or the first `heads` (Falcon's 71 q
// heads and its one k head).
template <int HD, bool QK>
__global__ void __launch_bounds__(256)
rope_kernel(uint16_t* __restrict__ qkv, long long ld, int heads, const int* __restrict__ cu_seqlens, int n_seq,
            const int* __restrict__ positions, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
            int max_pos) {
  static_assert(HD == 64 || HD == 128, "head_dim 64 or 128");
  constexpr int HP = HD / 4, HP_LOG2 = HD == 128 ? 5 : 4;  // pairs of adjacent j per head
  const long long tok = blockIdx.x;
  int pos;
  if (positions) {
    pos = positions[tok];
  } else {  // position inside its sequence: binary search of the packed offsets
    int lo = 0, hi = n_seq;  // cu_seqlens[lo] <= tok < cu_seqlens[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (cu_seqlens[mid] <= tok) lo = mid; else hi = mid;
    }
    pos = (int)(tok - cu_seqlens[lo]);
  }
  uint16_t* row = qkv + tok * ld;
  const int pairs = (QK ? 2 * heads : heads) * HP;  // rotated heads x HD / 4 pairs of adjacent j
  if (pos < 0 || pos >= max_pos) {  // outside the table: the row's q | k become NaN rather than a silent wrong result
    for (int p = threadIdx.x; p < pairs; p += blockDim.x) {
      const int hh = p >> HP_LOG2, j = (p & (HP - 1)) * 2;
      *reinterpret_cast<uint32_t*>(row + hh * HD + j) = 0x7e007e00u;
      *reinterpret_cast<uint32_t*>(row + hh * HD + HD / 2 + j) = 0x7e007e00u;
    }
    return;
  }
  const float2* cr = reinterpret_cast<const float2*>(cos_t + (long long)pos * (HD / 2));
  const float2* sr = reinterpret_cast<const float2*>(sin_t + (long long)pos * (HD / 2));
  for (int p = threadIdx.x; p < pairs; p += blockDim.x) {
    const int hh = p >> HP_LOG2, j = (p & (HP - 1)) * 2;
    uint32_t* a = reinterpret_cast<uint32_t*>(row + hh * HD + j);
    uint32_t* b = reinterpret_cast<uint32_t*>(row + hh * HD + HD / 2 + j);
    const float2 x1 = f16x2_to_float2(*a), x2 = f16x2_to_float2(*b);
    const float2 c = __ldg(cr + (j >> 1)), s = __ldg(sr + (j >> 1));
    *a = pack_f16x2(x1.x * c.x - x2.x * s.x, x1.y * c.y - x2.y * s.y);
    *b = pack_f16x2(x2.x * c.x + x1.x * s.x, x2.y * c.y + x1.y * s.y);
  }
}

// LlamaMLP's act_fn(gate_proj(y)) * up_proj(y) on the fused gate | up GEMM output: in fp32 [rows, 2 H],
// out fp16 [rows, H] (the operand of down_proj).  4 columns per thread.
__global__ void __launch_bounds__(256)
swiglu_f16_kernel(const float4* __restrict__ in, uint2* __restrict__ out, long long total4, int h4) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total4) return;
  const long long r = idx / h4;
  const int j = (int)(idx % h4);
  const float4 a = __ldcs(in + r * 2 * h4 + j), b = __ldcs(in + r * 2 * h4 + h4 + j);
  const float ox = a.x / (1.0f + expf(-a.x)) * b.x, oy = a.y / (1.0f + expf(-a.y)) * b.y;
  const float oz = a.z / (1.0f + expf(-a.z)) * b.z, ow = a.w / (1.0f + expf(-a.w)) * b.w;
  out[idx] = make_uint2(pack_f16x2(ox, oy), pack_f16x2(oz, ow));
}

}  // namespace

extern "C" int mer_rmsnorm(const float* x, const float* w, void* y16, float* acc, long long rows, int dim, float eps,
                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(x && w && (y16 || acc) && rows > 0, "mer_rmsnorm: bad arguments");
  MER_REQUIRE(rows < (1ll << 31), "mer_rmsnorm: %lld rows", rows);
  MER_REQUIRE(dim > 0 && dim % 256 == 0 && dim <= RMS_MAX_DIM, "mer_rmsnorm: dim %d (a multiple of 256 up to %d)", dim,
              RMS_MAX_DIM);
  rmsnorm_kernel<<<(unsigned)rows, RMS_THREADS, 0, stream>>>(x, w, static_cast<uint16_t*>(y16), acc, dim, eps);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_layernorm_f16(const float* x, const float* gamma, const float* beta, void* y16, float* y32, float* acc,
                                 long long rows, int dim, float eps, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(x && gamma && beta && (y16 || y32 || acc) && rows > 0, "mer_layernorm_f16: bad arguments");
  MER_REQUIRE(rows < (1ll << 31), "mer_layernorm_f16: %lld rows", rows);
  MER_REQUIRE(dim > 0 && dim % 256 == 0 && dim <= RMS_MAX_DIM, "mer_layernorm_f16: dim %d (a multiple of 256 up to %d)",
              dim, RMS_MAX_DIM);
  MER_REQUIRE(y32 != x, "mer_layernorm_f16: y32 may not alias x");
  layernorm_f16_kernel<false><<<(unsigned)rows, RMS_THREADS, 0, stream>>>(x, gamma, beta, static_cast<uint16_t*>(y16),
                                                                          y32, acc, dim, eps, 0);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_rope_f16(void* qkv16, long long ld, long long tokens, int heads, const int32_t* cu_seqlens,
                            int n_seq, const int32_t* positions, const float* cos_t, const float* sin_t, int max_pos,
                            void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(qkv16 && cos_t && sin_t && (positions || (cu_seqlens && n_seq > 0)),
              "mer_rope_f16: null operand");
  MER_REQUIRE(tokens > 0 && tokens < (1ll << 31) && heads > 0 && ld >= 2ll * heads * 128 && ld % 2 == 0 && max_pos > 0,
              "mer_rope_f16: bad shape (%lld tokens, %d heads, ld %lld)", tokens, heads, ld);
  rope_kernel<128, true><<<(unsigned)tokens, 256, 0, stream>>>(static_cast<uint16_t*>(qkv16), ld, heads, cu_seqlens,
                                                                n_seq, positions, cos_t, sin_t, max_pos);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_layernorm_ld_f16(const float* x, long long ld, const float* gamma, const float* beta, void* y16,
                                    float* y32, float* acc, long long rows, int dim, float eps, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(x && gamma && beta && (y16 || y32 || acc) && rows > 0, "mer_layernorm_ld_f16: bad arguments");
  MER_REQUIRE(rows < (1ll << 31), "mer_layernorm_ld_f16: %lld rows", rows);
  MER_REQUIRE(dim > 0 && dim % 64 == 0 && dim <= RMS_MAX_DIM, "mer_layernorm_ld_f16: dim %d (a multiple of 64 up to %d)",
              dim, RMS_MAX_DIM);
  MER_REQUIRE(ld >= dim && ld % 4 == 0, "mer_layernorm_ld_f16: row pitch %lld (a multiple of 4 >= dim %d)", ld, dim);
  MER_REQUIRE(y32 != x, "mer_layernorm_ld_f16: y32 may not alias x");
  layernorm_f16_kernel<true><<<(unsigned)rows, RMS_THREADS, 0, stream>>>(x, gamma, beta, static_cast<uint16_t*>(y16),
                                                                         y32, acc, dim, eps, ld);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_rope_hd_f16(void* qkv16, long long ld, long long tokens, int rot_heads, int head_dim,
                               const int32_t* cu_seqlens, int n_seq, const int32_t* positions, const float* cos_t,
                               const float* sin_t, int max_pos, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(head_dim == 64 || head_dim == 128, "mer_rope_hd_f16: head_dim %d (64 or 128)", head_dim);
  MER_REQUIRE(qkv16 && cos_t && sin_t && (positions || (cu_seqlens && n_seq > 0)), "mer_rope_hd_f16: null operand");
  MER_REQUIRE(tokens > 0 && tokens < (1ll << 31) && rot_heads > 0 && ld >= (long long)rot_heads * head_dim &&
                  ld % 2 == 0 && max_pos > 0,
              "mer_rope_hd_f16: bad shape (%lld tokens, %d heads of %d, ld %lld)", tokens, rot_heads, head_dim, ld);
  uint16_t* q = static_cast<uint16_t*>(qkv16);
  if (head_dim == 64)
    rope_kernel<64, false><<<(unsigned)tokens, 256, 0, stream>>>(q, ld, rot_heads, cu_seqlens, n_seq, positions, cos_t,
                                                                 sin_t, max_pos);
  else
    rope_kernel<128, false><<<(unsigned)tokens, 256, 0, stream>>>(q, ld, rot_heads, cu_seqlens, n_seq, positions,
                                                                  cos_t, sin_t, max_pos);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_swiglu_f16(const float* in, void* out16, long long rows, int hidden, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(in && out16 && rows > 0 && hidden > 0 && hidden % 4 == 0, "mer_swiglu_f16: bad arguments");
  const long long total4 = rows * (hidden / 4);
  swiglu_f16_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(in),
                                                                          static_cast<uint2*>(out16), total4,
                                                                          hidden / 4);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}
