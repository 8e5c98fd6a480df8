// rowwise.cu — HBM-bound row kernels: LayerNorm (+ optional "last-4 hidden states" accumulation)
// and the fp32 -> tf32 rounding pass used on weights at load time.
//
// LayerNorm follows torch.nn.LayerNorm exactly (biased variance, eps inside the sqrt), one warp
// per row, 128-bit loads/stores, the whole row kept in registers between the mean pass and the
// variance pass (two-pass, no E[x^2]-E[x]^2 cancellation).  Algorithmic traffic: 8 bytes per
// element (+4 per element for the accumulation buffer, +4 more when it is read back).
// Reference ops: HF ViTLayer.layernorm_before/after (modeling_vit.py:325-340),
// HubertEncoderLayer.layer_norm/final_layer_norm (modeling_hubert.py:372-405),
// BertSelfOutput/BertOutput.LayerNorm.
#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

template <int VEC>  // VEC float4 per lane: dim = 128 * VEC
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float* __restrict__ y, void* __restrict__ ys,
                 float* __restrict__ acc, long long rows, float eps, int flags) {
  constexpr int DIM = 128 * VEC;
  const int lane = threadIdx.x & 31;
  const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
  long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);

  float4 g[VEC], b[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    g[i] = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i);
    b[i] = __ldg(reinterpret_cast<const float4*>(beta) + lane + 32 * i);
  }
  for (; row < rows; row += warps_total) {
    const float4* xr = reinterpret_cast<const float4*>(x + row * DIM);
    float4 v[VEC];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      v[i] = xr[lane + 32 * i];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mean = warp_sum(s) * (1.0f / DIM);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
      q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
    }
    const float rstd = 1.0f / sqrtf(warp_sum(q) * (1.0f / DIM) + eps);
    const bool y16 = (flags & MER_LN_OUT_F16) != 0;  // y is an fp16 row (the F16 GEMM operand)
    float4* yr = (y && !y16) ? reinterpret_cast<float4*>(y + row * DIM) : nullptr;
    uint2* yh = (y && y16) ? reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(y) + row * DIM) : nullptr;
    const bool ys16 = (flags & MER_LN_SPLIT_F16) != 0;  // the second output is an fp16 row instead of a bf16 split row
    float* ysr = (ys && !ys16) ? reinterpret_cast<float*>(ys) + row * DIM : nullptr;  // split row: DIM 4-byte slots
    uint2* ysh = (ys && ys16) ? reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(ys) + row * DIM) : nullptr;
    float4* ar = acc ? reinterpret_cast<float4*>(acc + row * DIM) : nullptr;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      float4 o;
      o.x = v[i].x * rstd * g[i].x + b[i].x;
      o.y = v[i].y * rstd * g[i].y + b[i].y;
      o.z = v[i].z * rstd * g[i].z + b[i].z;
      o.w = v[i].w * rstd * g[i].w + b[i].w;
      if (flags & MER_LN_GELU) {
        o.x = gelu_erf_fast(o.x); o.y = gelu_erf_fast(o.y); o.z = gelu_erf_fast(o.z); o.w = gelu_erf_fast(o.w);
      }
      if (ar) {
        if (flags & MER_LN_ACC_INIT) {
          ar[lane + 32 * i] = o;
        } else if (flags & MER_LN_ACC_ADD) {
          float4 a = ar[lane + 32 * i];
          a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w;
          ar[lane + 32 * i] = a;
        }
      }
      if (ysr) store_split4(ysr, 4 * (lane + 32 * i), o);
      if (ysh) ysh[lane + 32 * i] = make_uint2(pack_f16x2(o.x, o.y), pack_f16x2(o.z, o.w));
      if (yh) yh[lane + 32 * i] = make_uint2(pack_f16x2(o.x, o.y), pack_f16x2(o.z, o.w));
      if (yr) {
        if (flags & MER_LN_ROUND_TF32) {
          o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w);
        }
        yr[lane + 32 * i] = o;
      }
    }
  }
}

// Round-2 form (default; MER_LN_VER=1 keeps the kernel above): the same arithmetic, row for row, with gamma / beta in
// shared memory instead of 2 x 4 VEC registers per lane.  The first form needs 96 registers -> two blocks = 16 warps
// per SM, each alternating between a load phase (3 KB in flight) and a reduce / store phase with nothing in flight.  Here a warp
// fits 64 registers at 768 columns (four blocks = 32 warps per SM) and requests its NEXT row before it reduces and stores the
// current one, so loads stay in flight through the whole loop.
// 1 / (the width the statistics run over): DIM, or the valid width of a padded row (MER_LN_PAD)
template <int DIM, typename... P>
__device__ __forceinline__ float ln_inv_width(P... valid) {
  if constexpr (sizeof...(P) == 0) return 1.0f / DIM;
  else return 1.0f / (float)(valid + ...);
}
// zero the elements of float4 slot `slot` (columns 4 slot .. 4 slot + 3) at or beyond column `valid`
__device__ __forceinline__ void zero_pad4(float4& v, int slot, int valid) {
  const int c = 4 * slot;
  if (c >= valid) v.x = 0.f;
  if (c + 1 >= valid) v.y = 0.f;
  if (c + 2 >= valid) v.z = 0.f;
  if (c + 3 >= valid) v.w = 0.f;
}

// valid: empty, or (MER_LN_PAD) one int, the valid width of rows padded to DIM: the statistics run over the first
// `valid` columns and every output is zero beyond them.  An empty pack keeps the unpadded instances' parameter list and
// code.
template <int VEC, typename... P>
__global__ void __launch_bounds__(256, VEC <= 6 ? 4 : VEC <= 8 ? 3 : 2)
layernorm2_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                  const float* __restrict__ beta, float* __restrict__ y, void* __restrict__ ys,
                  float* __restrict__ acc, long long rows, float eps, int flags, P... valid) {
  constexpr int DIM = 128 * VEC;
  constexpr bool PAD = sizeof...(P) > 0;
  __shared__ float4 gs[32 * VEC], bs[32 * VEC];
  for (int i = threadIdx.x; i < 32 * VEC; i += blockDim.x) {
    gs[i] = __ldg(reinterpret_cast<const float4*>(gamma) + i);
    bs[i] = __ldg(reinterpret_cast<const float4*>(beta) + i);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
  long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const bool y16 = (flags & MER_LN_OUT_F16) != 0;   // y is an fp16 row (the F16 GEMM operand)
  const bool ys16 = (flags & MER_LN_SPLIT_F16) != 0;  // the second output is an fp16 row instead of a bf16 split row
  float4 v[VEC];
  {
    const float4* xr = reinterpret_cast<const float4*>(x + row * DIM);
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = xr[lane + 32 * i];
  }
  for (; row < rows; row += warps_total) {
    if constexpr (PAD) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) zero_pad4(v[i], lane + 32 * i, (valid + ...));
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) * ln_inv_width<DIM>(valid...);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
      if constexpr (PAD) zero_pad4(v[i], lane + 32 * i, (valid + ...));
      q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
    }
    const float rstd = 1.0f / sqrtf(warp_sum(q) * ln_inv_width<DIM>(valid...) + eps);
    float4* yr = (y && !y16) ? reinterpret_cast<float4*>(y + row * DIM) : nullptr;
    uint2* yh = (y && y16) ? reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(y) + row * DIM) : nullptr;
    float* ysr = (ys && !ys16) ? reinterpret_cast<float*>(ys) + row * DIM : nullptr;  // split row: DIM 4-byte slots
    uint2* ysh = (ys && ys16) ? reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(ys) + row * DIM) : nullptr;
    float4* ar = acc ? reinterpret_cast<float4*>(acc + row * DIM) : nullptr;
    // (y == x is allowed: a warp has its whole row in registers before it writes; the NEXT row belongs to this warp too)
    const long long nrow = row + warps_total;
    const float4* xn = reinterpret_cast<const float4*>(x + (nrow < rows ? nrow : row) * DIM);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float4 g = gs[lane + 32 * i], b = bs[lane + 32 * i];
      float4 o;
      o.x = v[i].x * rstd * g.x + b.x;
      o.y = v[i].y * rstd * g.y + b.y;
      o.z = v[i].z * rstd * g.z + b.z;
      o.w = v[i].w * rstd * g.w + b.w;
      v[i] = xn[lane + 32 * i];  // the next row's slot i: in flight while this row is finished and stored
      if (flags & MER_LN_GELU) {
        o.x = gelu_erf_fast(o.x); o.y = gelu_erf_fast(o.y); o.z = gelu_erf_fast(o.z); o.w = gelu_erf_fast(o.w);
      }
      if constexpr (PAD) zero_pad4(o, lane + 32 * i, (valid + ...));
      if (ar) {
        if (flags & MER_LN_ACC_INIT) {
          ar[lane + 32 * i] = o;
        } else if (flags & MER_LN_ACC_ADD) {
          float4 a = ar[lane + 32 * i];
          a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w;
          if constexpr (PAD) zero_pad4(a, lane + 32 * i, (valid + ...));
          ar[lane + 32 * i] = a;
        }
      }
      if (ysr) store_split4(ysr, 4 * (lane + 32 * i), o);
      if (ysh) ysh[lane + 32 * i] = make_uint2(pack_f16x2(o.x, o.y), pack_f16x2(o.z, o.w));
      if (yh) yh[lane + 32 * i] = make_uint2(pack_f16x2(o.x, o.y), pack_f16x2(o.z, o.w));
      if (yr) {
        if (flags & MER_LN_ROUND_TF32) {
          o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w);
        }
        yr[lane + 32 * i] = o;
      }
    }
  }
}

// fp32 [rows,K] -> split bf16 rows (128-byte groups of 32 hi | 32 lo), K % 32 == 0
__global__ void split_bf16_kernel(const float* __restrict__ in, void* __restrict__ out, long long rows,
                                  int K) {
  const long long total = rows * (K / 4);
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < total; i += stride) {
    const long long r = i / (K / 4);
    const int c4 = (int)(i % (K / 4));
    const float4 v = *reinterpret_cast<const float4*>(in + r * K + c4 * 4);
    store_split4(reinterpret_cast<float*>(out) + r * K, c4 * 4, v);
  }
}

// fp32 -> fp16 (round-to-nearest, saturating), 4 elements per thread
__global__ void cast_f16_kernel(const float4* __restrict__ in, uint2* __restrict__ out, long long n4) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n4; i += stride) {
    const float4 v = in[i];
    out[i] = make_uint2(pack_f16x2(v.x, v.y), pack_f16x2(v.z, v.w));
  }
}

// acc = x (init) or acc += x, float4-wise
__global__ void accumulate_kernel(const float4* __restrict__ x, float4* __restrict__ acc, long long n4, int init) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n4; i += stride) {
    float4 v = x[i];
    if (!init) {
      const float4 a = acc[i];
      v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    }
    acc[i] = v;
  }
}

__global__ void round_tf32_kernel(float* x, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) x[i] = round_tf32(x[i]);
}

}  // namespace

int mer_layernorm_launch(const float* x, const float* gamma, const float* beta, float* y,
                         void* y_split, float* acc, long long rows, int dim, float eps, int flags,
                         cudaStream_t stream) {
  MER_REQUIRE(x && gamma && beta && (y || y_split), "mer_layernorm: null operand");
  // y == x and y_split == x are both fine: a warp holds its whole row in registers before it
  // writes, and a split row occupies exactly the bytes of the fp32 row it replaces.  (An fp16 y must
  // not alias x: its rows are half as long.)
  MER_REQUIRE(!((flags & MER_LN_OUT_F16) && (const void*)y == (const void*)x),
              "mer_layernorm: an fp16 output cannot alias the input");
  // MER_LN_PAD: dim is the valid width of rows padded to the next multiple of 128
  const bool pad = (flags & MER_LN_PAD) != 0;
  const int width = pad ? (dim + 127) / 128 * 128 : dim;
  MER_REQUIRE(dim > 0 && (width == 768 || width == 512 || width == 1024 || width == 1280 || width == 1536 ||
                          width == 128 || width == 384 || width == 256),
              "mer_layernorm: dim %d not supported (512, 768, 1024, 1280, 1536) (also 128, 384 and 256; with MER_LN_PAD, "
              "a valid width whose next multiple of 128 is one of these)", dim);
  if (rows <= 0) return 0;
  const int warps_per_block = 8;
  long long blocks = (rows + warps_per_block - 1) / warps_per_block;
  const long long max_blocks = (long long)mer_num_sms() * 16;
  if (blocks > max_blocks) blocks = max_blocks;
  // algorithmic bytes: the fp32 row in, each output row (fp16: 2 B/elem), the accumulator (write, or read+write)
  const double out_b = (y ? ((flags & MER_LN_OUT_F16) ? 2.0 : 4.0) : 0.0) + (y_split ? 4.0 : 0.0) +
                       (acc ? ((flags & MER_LN_ACC_ADD) ? 8.0 : 4.0) : 0.0);
  const int prof = mer_prof_begin(MER_PROF_LAYERNORM, (double)rows * width * (4.0 + out_b), stream);
  const char* ver = getenv("MER_LN_VER");  // read at every launch: tests run both forms in one process
  const bool v1 = ver && atoi(ver) == 1;
#define MER_LN_LAUNCH(VEC)                                                                                          \
  do {                                                                                                              \
    if (pad) layernorm2_kernel<VEC, int><<<(int)blocks, 256, 0, stream>>>(x, gamma, beta, y, y_split, acc, rows, eps,  \
                                                                         flags, dim);                                 \
    else if (v1) layernorm_kernel<VEC><<<(int)blocks, 256, 0, stream>>>(x, gamma, beta, y, y_split, acc, rows, eps,   \
                                                                        flags);                                       \
    else layernorm2_kernel<VEC><<<(int)blocks, 256, 0, stream>>>(x, gamma, beta, y, y_split, acc, rows, eps, flags);    \
  } while (0)
  if (width == 768) MER_LN_LAUNCH(6);
  else if (width == 1024) MER_LN_LAUNCH(8);
  else if (width == 1280) MER_LN_LAUNCH(10);  // whisper-large-v2
  else if (width == 1536) MER_LN_LAUNCH(12);  // dinov2-giant
  else if (width == 128) MER_LN_LAUNCH(1);    // ALBERT's embedding LayerNorm
  else if (width == 384) MER_LN_LAUNCH(3);    // albert_chinese_small; albert_chinese_tiny's 312 padded to 384
  else if (width == 256) MER_LN_LAUNCH(2);    // ELECTRA-small / LERT-small (hidden 256)
  else MER_LN_LAUNCH(4);
#undef MER_LN_LAUNCH
  mer_prof_end(prof, stream);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_accumulate_launch(const float* x, float* acc, long long n, int init, cudaStream_t stream) {
  MER_REQUIRE(x && acc && n % 4 == 0, "mer_accumulate: bad operands");
  if (n <= 0) return 0;
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > mer_num_sms() * 32) blocks = mer_num_sms() * 32;
  accumulate_kernel<<<(int)blocks, 256, 0, stream>>>(reinterpret_cast<const float4*>(x),
                                                     reinterpret_cast<float4*>(acc), n / 4, init);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_cast_f16_launch(const float* in, void* out, long long n, cudaStream_t stream) {
  MER_REQUIRE(in && out && n % 4 == 0, "mer_cast_f16: bad operands");
  if (n <= 0) return 0;
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > mer_num_sms() * 32) blocks = mer_num_sms() * 32;
  cast_f16_kernel<<<(int)blocks, 256, 0, stream>>>(reinterpret_cast<const float4*>(in),
                                                   reinterpret_cast<uint2*>(out), n / 4);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_round_tf32(float* x, long long n, void* stream) {
  if (n <= 0) return 0;
  long long blocks = (n + 255) / 256;
  if (blocks > mer_num_sms() * 32) blocks = mer_num_sms() * 32;
  round_tf32_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, n);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_split_bf16(const float* in, void* out, long long rows, int K, void* stream) {
  MER_REQUIRE(in && out && (const void*)in != out && K > 0 && K % 32 == 0, "mer_split_bf16: bad operands");
  if (rows <= 0) return 0;
  long long blocks = (rows * (K / 4) + 255) / 256;
  if (blocks > mer_num_sms() * 32) blocks = mer_num_sms() * 32;
  split_bf16_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(in, out, rows, K);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}
