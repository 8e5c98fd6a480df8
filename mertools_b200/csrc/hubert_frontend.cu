// hubert_frontend.cu — the HBM-bound head of the audio encoder (SURVEY.md kernel rows A0/A1):
//
//   wave_normalize   : HF Wav2Vec2FeatureExtractor zero-mean / unit-variance, eps 1e-7
//                      (feature_extraction_wav2vec2.py:78-97, called at
//                      extract_audio_huggingface.py:94)
//   conv0_moments    : per clip, the 10 tap sums and 55 tap products of the waveform at stride 5, in double
//   conv0_coef       : ... turned into each channel's GroupNorm(512 groups) mean and gamma / sqrt(var + eps)
//                      (modeling_hubert.py:154-175) -- conv0 is linear, so its statistics follow from the moments
//   conv0_apply      : compute conv0 = Conv1d(1->512, k=10, s=5), normalise, affine, exact GELU, write the
//                      TIME-MAJOR activation [B, T0_pad, 512] that the conv1 implicit GEMM reads (split bf16
//                      hi|lo rows for the BF16X3 GEMM, or tf32-rounded fp32).
//
// The fp32 conv0 output (32.8 MB per 5 s clip) is never materialised un-normalised, and it is computed ONCE: the
// waveform (320 KB per clip) is read three times (normalise, moments, apply).  Algorithmic traffic per clip:
// 3 x 320 KB in + 15,999 x 512 x 4 B = 32.8 MB out.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int C0 = 512;
constexpr int K0 = 10;
constexpr int S0 = 5;

__device__ __forceinline__ double block_sum_double(double v, double* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  double r = 0.0;
  const int nw = blockDim.x >> 5;
  for (int i = 0; i < nw; ++i) r += sh[i];
  __syncthreads();
  return r;
}

// one block per clip; two passes over the waveform (mean, then variance about the mean)
__global__ void __launch_bounds__(1024)
wave_normalize_kernel(const float* __restrict__ in, float* __restrict__ out, int L, long long ld_in,
                      long long ld_out) {
  __shared__ double sh[32];
  const float* x = in + (long long)blockIdx.x * ld_in;
  float* y = out + (long long)blockIdx.x * ld_out;
  double s = 0.0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) s += (double)x[i];
  const double mean = block_sum_double(s, sh) / (double)L;
  double q = 0.0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const double d = (double)x[i] - mean;
    q += d * d;
  }
  const double var = block_sum_double(q, sh) / (double)L;
  const float meanf = (float)mean;
  const float denom = sqrtf((float)var + 1e-7f);
  for (int i = threadIdx.x; i < L; i += blockDim.x) y[i] = (x[i] - meanf) / denom;
}

// ragged batch: row b holds lengths[b] samples (statistics over those), the rest of the row is written as zeros
__global__ void __launch_bounds__(1024)
wave_normalize_ragged_kernel(const float* __restrict__ in, float* __restrict__ out, const int* __restrict__ lengths,
                             int L, long long ld_in, long long ld_out) {
  __shared__ double sh[32];
  const float* x = in + (long long)blockIdx.x * ld_in;
  float* y = out + (long long)blockIdx.x * ld_out;
  const int n = lengths[blockIdx.x];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += (double)x[i];
  const double mean = block_sum_double(s, sh) / (double)n;
  double q = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double d = (double)x[i] - mean;
    q += d * d;
  }
  const double var = block_sum_double(q, sh) / (double)n;
  const float meanf = (float)mean;
  const float denom = sqrtf((float)var + 1e-7f);
  for (int i = threadIdx.x; i < L; i += blockDim.x) y[i] = i < n ? (x[i] - meanf) / denom : 0.f;
}

// ---- GroupNorm statistics of conv0 WITHOUT a pass over its output ----
// conv0 is linear in the waveform: y[t, c] = sum_k w[c, k] x[5 t + k].  So, per clip,
//     sum_t y[t, c]   = sum_k w[c, k] X_k,                  X_k    = sum_t x[5 t + k]
//     sum_t y[t, c]^2 = sum_{k, k'} w[c, k] w[c, k'] R_kk',  R_kk' = sum_t x[5 t + k] x[5 t + k']
// i.e. the statistics of all 512 channels follow from 10 tap sums and the 10 x 10 (symmetric: 55 entries) tap
// correlation matrix of the clip.  Round 1 / early round 2 recomputed the whole convolution in a statistics pass
// (half of the kernel's arithmetic; the kernel is ALU-bound); now `conv0_moments_kernel` accumulates the 65 moments in
// double (products of the fp32 samples are exact in double) and `conv0_coef_kernel` turns them into the per-(clip,
// channel) mean and gamma / sqrt(var + eps) that the apply kernel uses -- the statistics of the EXACT convolution
// output, within 1e-7 (relative, variance) of those of the fp32-rounded one the reference normalises with.
constexpr int NMOM = 65;       // 10 tap sums + 55 products (k <= k')
constexpr int MOM_LD = 72;     // doubles per clip in the moments buffer
constexpr int MCHUNK = 1024;   // frames per block of the moments kernel
constexpr int MOM_THREADS = 288;  // 65 moments x 4 frame phases = 260 working threads

// RAGGED: clip b has t0s[b] <= T0 frames: the moments run over those.
template <bool RAGGED>
__global__ void __launch_bounds__(MOM_THREADS)
conv0_moments_kernel(const float* __restrict__ wave, long long ld_wave, int T0, double* __restrict__ mom /*[B, MOM_LD]*/,
                     const int* __restrict__ t0s) {
  __shared__ float xs[MCHUNK * S0 + K0];
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * MCHUNK;
  if (RAGGED) T0 = t0s[b];
  if (t0 >= T0) return;  // block-uniform
  const int nt = min(MCHUNK, T0 - t0);
  const float* x = wave + (long long)b * ld_wave + (long long)t0 * S0;
  const int nx = (nt - 1) * S0 + K0;
  for (int i = threadIdx.x; i < nx; i += blockDim.x) xs[i] = x[i];
  __syncthreads();
  const int p = threadIdx.x >> 2, ph = threadIdx.x & 3;
  if (p >= NMOM) return;  // (the last warp's tail; no barrier follows)
  int k = p, k2 = -1;     // p < 10: tap sum k
  if (p >= K0) {          // p - 10 enumerates the pairs (k, k2), k <= k2, row by row
    int q = p - K0;
    k = 0;
    while (q >= K0 - k) { q -= K0 - k; ++k; }
    k2 = k + q;
  }
  double acc = 0.0;
  if (k2 < 0) {
    for (int t = ph; t < nt; t += 4) acc += (double)xs[t * S0 + k];
  } else {
    for (int t = ph; t < nt; t += 4) acc = fma((double)xs[t * S0 + k], (double)xs[t * S0 + k2], acc);
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);  // the four frame phases sit in adjacent lanes
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  if (ph == 0) atomicAdd(&mom[(long long)b * MOM_LD + p], acc);
}

// grid B, 512 threads (one channel each): moments -> (mean, gamma / sqrt(var + 1e-5)) as floats.
// GroupNorm with num_groups == channels: biased variance over time, eps 1e-5 (modeling_hubert.py:154-175).
__global__ void __launch_bounds__(C0)
conv0_coef_kernel(const double* __restrict__ mom, const float* __restrict__ w0, const float* __restrict__ gamma, int T0,
                  const int* __restrict__ t0s, float2* __restrict__ coef /*[B, 512]*/) {
  __shared__ double m[NMOM];
  const int b = blockIdx.x, c = threadIdx.x;
  if (c < NMOM) m[c] = mom[(long long)b * MOM_LD + c];
  __syncthreads();
  if (t0s) T0 = t0s[b];
  double w[K0];
#pragma unroll
  for (int k = 0; k < K0; ++k) w[k] = (double)__ldg(w0 + c * K0 + k);
  double s = 0.0, q = 0.0;
  int idx = K0;
#pragma unroll
  for (int k = 0; k < K0; ++k) {
    s = fma(w[k], m[k], s);
#pragma unroll
    for (int k2 = k; k2 < K0; ++k2, ++idx) q = fma((k2 == k ? 1.0 : 2.0) * w[k] * w[k2], m[idx], q);
  }
  const double mean_d = s / (double)T0;
  double var_d = q / (double)T0 - mean_d * mean_d;
  if (var_d < 0.0) var_d = 0.0;
  coef[(long long)b * C0 + c] = make_float2((float)mean_d, __ldg(gamma + c) * (float)(1.0 / sqrt(var_d + 1e-5)));
}

// grid (chunks, B); each block covers TCHUNK output frames.
constexpr int TCHUNK = 128;

// one channel per thread (512 threads): the plain form (tf32-rounded fp32 output, or MER_CONV0_PACKED=0)
__global__ void __launch_bounds__(C0)
conv0_apply_kernel(const float* __restrict__ wave, long long ld_wave, const float* __restrict__ w0,
                   const float* __restrict__ beta, const float2* __restrict__ coef, int T0,
                   long long out_bstride /*floats*/, int split_out, float* __restrict__ out) {
  __shared__ float xs[TCHUNK * S0 + K0];
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * TCHUNK;
  const int nt = min(TCHUNK, T0 - t0);  // ragged batches: frames past the clip's own count are still written (finite, unused)
  const float* x = wave + (long long)b * ld_wave + (long long)t0 * S0;
  const int nx = (nt - 1) * S0 + K0;
  for (int i = threadIdx.x; i < nx; i += blockDim.x) xs[i] = x[i];
  __syncthreads();
  const int c = threadIdx.x;
  float w[K0];
#pragma unroll
  for (int k = 0; k < K0; ++k) w[k] = __ldg(w0 + c * K0 + k);
  const float2 mg = coef[(long long)b * C0 + c];
  const float mean = mg.x, g = mg.y;
  const float bt = __ldg(beta + c);
  float* orow = out + (long long)b * out_bstride + (long long)t0 * C0;
  for (int t = 0; t < nt; ++t) {
    float y = 0.f;
#pragma unroll
    for (int k = 0; k < K0; ++k) y = fmaf(w[k], xs[t * S0 + k], y);
    const float v = gelu_erf_fast((y - mean) * g + bt);
    if (split_out == 2) reinterpret_cast<__half*>(out)[((long long)b * out_bstride + (long long)(t0 + t) * C0) + c] = __float2half_rn(v);
    else if (split_out) store_split1(orow + (long long)t * C0, c, v);
    else orow[(long long)t * C0 + c] = round_tf32(v);
  }
}

// The default form (split-bf16 output): two adjacent channels per thread on the packed fp32 pipe (FFMA2 with the sample
// as a broadcast operand), FOUR frames per iteration sharing one window of 25 samples (six 16-byte shared-memory loads
// and one scalar instead of 40 scalar loads: 5 t is a multiple of 4 floats when t is a multiple of 4), the packed GELU,
// 4 + 4 byte split stores.  Per channel the conv arithmetic is the same sequence of fma.rn as the scalar kernel.
// F16: the row is 512 fp16 values (the MER_GEMM_F16 operand: conv1 on fp16 operands); else a split-bf16 row
template <bool F16>
__device__ __forceinline__ void conv0_emit2(uint64_t y, uint64_t nmean2, uint64_t g2, uint64_t bt2, float* orow, int c) {
  float a0, a1, v0, v1;
  unpack2(fma2(add2(y, nmean2), g2, bt2), a0, a1);
  gelu_erf_fast2(a0, a1, v0, v1);
  if (F16) reinterpret_cast<uint32_t*>(orow)[c >> 1] = pack_f16x2(v0, v1);
  else store_split2(orow, c, v0, v1);
}

template <bool F16>
__global__ void __launch_bounds__(C0 / 2)
conv0_apply2_kernel(const float* __restrict__ wave, long long ld_wave, const float* __restrict__ w0,
                    const float* __restrict__ beta, const float2* __restrict__ coef, int T0,
                    long long out_bstride /*elements*/, float* __restrict__ out /*split bf16 rows, or fp16 rows*/) {
  __shared__ __align__(16) float xs[TCHUNK * S0 + K0 + 2];
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * TCHUNK;
  const int nt = min(TCHUNK, T0 - t0);
  const float* x = wave + (long long)b * ld_wave + (long long)t0 * S0;
  const int nx = (nt - 1) * S0 + K0;
  for (int i = threadIdx.x; i < TCHUNK * S0 + K0 + 2; i += blockDim.x) xs[i] = i < nx ? x[i] : 0.f;
  __syncthreads();
  const int c = 2 * threadIdx.x;
  uint64_t w[K0];
#pragma unroll
  for (int k = 0; k < K0; ++k) w[k] = pack2(__ldg(w0 + c * K0 + k), __ldg(w0 + (c + 1) * K0 + k));
  const float4 mg = *reinterpret_cast<const float4*>(coef + (long long)b * C0 + c);  // (mean, g) of c and c + 1
  const uint64_t nmean2 = pack2(-mg.x, -mg.z), g2 = pack2(mg.y, mg.w);
  const uint64_t bt2 = pack2(__ldg(beta + c), __ldg(beta + c + 1));
  // a row is C0 4-byte slots (split) or C0 2-byte values (fp16): address it in floats either way
  constexpr int RF = F16 ? C0 / 2 : C0;  // floats per row
  float* orow = out + ((long long)b * out_bstride + (long long)t0 * C0) / (F16 ? 2 : 1);
  int t = 0;
  for (; t + 4 <= nt; t += 4) {
    uint64_t xp[4 * S0 + K0 - S0];  // 25 samples, each as a (v, v) pair
    const float4* xv = reinterpret_cast<const float4*>(xs + t * S0);
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      const float4 v = xv[i];
      xp[4 * i + 0] = pack2(v.x, v.x); xp[4 * i + 1] = pack2(v.y, v.y);
      xp[4 * i + 2] = pack2(v.z, v.z); xp[4 * i + 3] = pack2(v.w, v.w);
    }
    {
      const float v = xs[t * S0 + 24];
      xp[24] = pack2(v, v);
    }
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      uint64_t y = pack2(0.f, 0.f);
#pragma unroll
      for (int k = 0; k < K0; ++k) y = fma2(w[k], xp[f * S0 + k], y);
      conv0_emit2<F16>(y, nmean2, g2, bt2, orow + (long long)(t + f) * RF, c);
    }
  }
  for (; t < nt; ++t) {
    uint64_t y = pack2(0.f, 0.f);
#pragma unroll
    for (int k = 0; k < K0; ++k) {
      const float xv = xs[t * S0 + k];
      y = fma2(w[k], pack2(xv, xv), y);
    }
    conv0_emit2<F16>(y, nmean2, g2, bt2, orow + (long long)t * RF, c);
  }
}

// conv0 (k = 10, stride 5, + bias) -> LayerNorm over the 512 channels -> GELU, the first layer of the
// feat_extract_norm="layer" feature encoder (HF HubertLayerNormConvLayer; hubert-large family).
// One warp = LN_ROWS consecutive frames; lane owns channels lane + 32 j (j < 16), weights transposed in
// smem ([tap][channel]: conflict-free), two-pass LayerNorm in registers via warp shuffles.
constexpr int LN_ROWS = 4;
__global__ void __launch_bounds__(256)
conv0_ln_kernel(const float* __restrict__ wave, long long ld_wave, const float* __restrict__ w0,
                const float* __restrict__ bias, const float* __restrict__ gamma, const float* __restrict__ beta,
                int T0, long long out_bstride, float* __restrict__ out) {
  __shared__ float ws[K0][C0];  // 20 KB
  __shared__ float xs[8][LN_ROWS * S0 + K0];
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < C0 * K0; i += blockDim.x) ws[i % K0][i / K0] = __ldg(w0 + i);
  __syncthreads();
  const int t0 = (blockIdx.x * 8 + warp) * LN_ROWS;
  if (t0 >= T0) return;
  const int nt = min(LN_ROWS, T0 - t0);
  const float* x = wave + (long long)b * ld_wave + (long long)t0 * S0;
  for (int i = lane; i < (nt - 1) * S0 + K0; i += 32) xs[warp][i] = x[i];
  __syncwarp();
  float acc[LN_ROWS][16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float bj = bias ? __ldg(bias + lane + 32 * j) : 0.f;
#pragma unroll
    for (int r = 0; r < LN_ROWS; ++r) acc[r][j] = bj;
  }
#pragma unroll
  for (int k = 0; k < K0; ++k) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float w = ws[k][lane + 32 * j];
#pragma unroll
      for (int r = 0; r < LN_ROWS; ++r) acc[r][j] = fmaf(w, xs[warp][r * S0 + k], acc[r][j]);
    }
  }
#pragma unroll
  for (int r = 0; r < LN_ROWS; ++r) {
    if (r >= nt) break;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) s += acc[r][j];
    const float mean = warp_sum(s) * (1.0f / C0);
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      acc[r][j] -= mean;
      q += acc[r][j] * acc[r][j];
    }
    const float rstd = 1.0f / sqrtf(warp_sum(q) * (1.0f / C0) + 1e-5f);
    float* orow = out + (long long)b * out_bstride + (long long)(t0 + r) * C0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = lane + 32 * j;
      const float v = gelu_erf_fast(acc[r][j] * rstd * __ldg(gamma + c) + __ldg(beta + c));
      store_split1(orow, c, v);
    }
  }
}

}  // namespace

int mer_wave_normalize_launch(const float* in, float* out, int B, int L, long long ld_in,
                              long long ld_out, cudaStream_t stream, const int* lengths) {
  MER_REQUIRE(in && out && B > 0 && L > 0, "mer_wave_normalize: bad arguments");
  // a pitch below the row length would make row b + 1 start inside row b: the rows' outputs would overwrite each other
  MER_REQUIRE(ld_in >= L && ld_out >= L, "mer_wave_normalize: row pitches %lld / %lld shorter than the %d samples of a row",
              ld_in, ld_out, L);
  if (lengths)
    wave_normalize_ragged_kernel<<<B, 1024, 0, stream>>>(in, out, lengths, L, ld_in, ld_out);
  else
    wave_normalize_kernel<<<B, 1024, 0, stream>>>(in, out, L, ld_in, ld_out);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_hubert_conv0_launch(const float* wave, long long ld_wave, int B, int L, const float* w0,
                            const float* gamma, const float* beta, double* stats, float* out,
                            long long out_bstride, int split_out, cudaStream_t stream, const int* t0s) {
  const int T0 = (L - K0) / S0 + 1;
  MER_REQUIRE(T0 > 0, "mer_hubert_conv0: waveform too short (%d samples)", L);
  // `stats` ([B, 512, 2] doubles as sized by the workspace plan) holds the moments [B, MOM_LD] doubles, then -- from
  // double B * 128 on -- the coefficients [B, 512] float2
  static_assert(MOM_LD <= 128, "moments and coefficients share the statistics buffer");
  double* mom = stats;
  float2* coef = reinterpret_cast<float2*>(stats + (size_t)B * 128);
  MER_CUDA_CHECK(cudaMemsetAsync(mom, 0, (size_t)B * MOM_LD * sizeof(double), stream));
  // algorithmic bytes: the waveform in twice (moments, apply), the [T0, 512] operand (4 B per element) out once
  const int prof = mer_prof_begin(MER_PROF_CONV0, (double)B * (2.0 * L * 4.0 + (double)T0 * C0 * (split_out == 2 ? 2.0 : 4.0)),
                                  stream);
  dim3 mgrid((T0 + MCHUNK - 1) / MCHUNK, B);
  if (t0s) conv0_moments_kernel<true><<<mgrid, MOM_THREADS, 0, stream>>>(wave, ld_wave, T0, mom, t0s);
  else conv0_moments_kernel<false><<<mgrid, MOM_THREADS, 0, stream>>>(wave, ld_wave, T0, mom, nullptr);
  MER_CUDA_CHECK(cudaGetLastError());
  conv0_coef_kernel<<<B, C0, 0, stream>>>(mom, w0, gamma, T0, t0s, coef);
  MER_CUDA_CHECK(cudaGetLastError());
  dim3 grid((T0 + TCHUNK - 1) / TCHUNK, B);
  const char* pk = getenv("MER_CONV0_PACKED");  // read at every launch: tests run both forms in one process
  if (!(pk && atoi(pk) == 0) && split_out == 2)  // fp16 rows (conv1 on fp16 operands)
    conv0_apply2_kernel<true><<<grid, C0 / 2, 0, stream>>>(wave, ld_wave, w0, beta, coef, T0, out_bstride, out);
  else if (!(pk && atoi(pk) == 0) && split_out)  // default; MER_CONV0_PACKED=0: one channel per thread
    conv0_apply2_kernel<false><<<grid, C0 / 2, 0, stream>>>(wave, ld_wave, w0, beta, coef, T0, out_bstride, out);
  else
    conv0_apply_kernel<<<grid, C0, 0, stream>>>(wave, ld_wave, w0, beta, coef, T0, out_bstride, split_out, out);
  mer_prof_end(prof, stream);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(3);
  return 0;
}

// ragged batch helpers: clip b occupies rows [b * Tmax, b * Tmax + tb[b]) of a padded [B, Tmax, dim] activation
__global__ void __launch_bounds__(256)
zero_tail_rows_f16_kernel(uint4* __restrict__ x, const int* __restrict__ tb, int Tmax, int dim8) {
  const int b = blockIdx.y;
  const long long n = (long long)(Tmax - tb[b]) * dim8;  // 16-byte slots of the clip's tail rows
  uint4* tail = x + ((long long)b * Tmax + tb[b]) * dim8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    tail[i] = make_uint4(0u, 0u, 0u, 0u);
}

__global__ void __launch_bounds__(256)
pack_rows_kernel(const float4* __restrict__ padded, const int* __restrict__ cu, int Tmax, int dim4,
                 float4* __restrict__ packed) {
  const int b = blockIdx.y;
  const long long n = (long long)(cu[b + 1] - cu[b]) * dim4;
  const float4* src = padded + (long long)b * Tmax * dim4;
  float4* dst = packed + (long long)cu[b] * dim4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = src[i];
}

int mer_zero_tail_rows_f16_launch(void* x16, const int* tb, int B, int Tmax, int dim, cudaStream_t stream) {
  MER_REQUIRE(x16 && tb && B > 0 && Tmax > 0 && dim % 8 == 0, "mer_zero_tail_rows_f16: bad operands");
  zero_tail_rows_f16_kernel<<<dim3(32, B), 256, 0, stream>>>(static_cast<uint4*>(x16), tb, Tmax, dim / 8);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_pack_rows_launch(const float* padded, const int* cu, int B, int Tmax, int dim, float* packed,
                         cudaStream_t stream) {
  MER_REQUIRE(padded && cu && packed && padded != packed && B > 0 && dim % 4 == 0, "mer_pack_rows: bad operands");
  pack_rows_kernel<<<dim3(32, B), 256, 0, stream>>>(reinterpret_cast<const float4*>(padded), cu, Tmax, dim / 4,
                                                    reinterpret_cast<float4*>(packed));
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_hubert_conv0_ln_launch(const float* wave, long long ld_wave, int B, int L, const float* w0,
                               const float* bias, const float* gamma, const float* beta, float* out,
                               long long out_bstride, cudaStream_t stream) {
  const int T0 = (L - K0) / S0 + 1;
  MER_REQUIRE(T0 > 0, "mer_hubert_conv0_ln: waveform too short (%d samples)", L);
  dim3 grid((T0 + 8 * LN_ROWS - 1) / (8 * LN_ROWS), B);
  conv0_ln_kernel<<<grid, 256, 0, stream>>>(wave, ld_wave, w0, bias, gamma, beta, T0, out_bstride, out);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_wave_normalize(const float* in, float* out, int batch, int n_samples,
                                  long long ld_in, long long ld_out, void* stream) {
  return mer_wave_normalize_launch(in, out, batch, n_samples, ld_in, ld_out,
                                   static_cast<cudaStream_t>(stream));
}

extern "C" int mer_hubert_conv0(const MerHubertModel* model, const float* wave, int batch, int n_samples,
                                long long ld_wave, const int* frames, int out_format, void* out, long long out_bstride,
                                void* workspace, long long workspace_bytes, void* stream) {
  MER_REQUIRE(model && wave && out && batch > 0 && model->conv0_w, "mer_hubert_conv0: bad arguments");
  const int T0 = n_samples >= K0 ? (n_samples - K0) / S0 + 1 : 0;
  MER_REQUIRE(T0 > 0, "mer_hubert_conv0: waveform too short (%d samples)", n_samples);
  MER_REQUIRE(ld_wave >= n_samples, "mer_hubert_conv0: row pitch %lld shorter than the %d samples of a row", ld_wave,
              n_samples);
  MER_REQUIRE(out_bstride >= (long long)T0 * C0, "mer_hubert_conv0: output batch stride %lld shorter than %d rows of %d",
              out_bstride, T0, C0);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (model->feat_norm_layer) {
    MER_REQUIRE(out_format == MER_EPI_SPLIT_BF16, "mer_hubert_conv0: the LayerNorm family writes split-bf16 rows only");
    MER_REQUIRE(model->conv_ln_g[0] && model->conv_ln_b[0], "mer_hubert_conv0: LayerNorm affine missing");
    return mer_hubert_conv0_ln_launch(wave, ld_wave, batch, n_samples, model->conv0_w, model->conv_b[0],
                                      model->conv_ln_g[0], model->conv_ln_b[0], static_cast<float*>(out), out_bstride, s);
  }
  MER_REQUIRE(out_format == MER_EPI_SPLIT_BF16 || (out_format == MER_EPI_OUT_F16 && out_bstride % 2 == 0),
              "mer_hubert_conv0: output format %d (split-bf16 = %d, or fp16 = %d with an even batch stride)", out_format,
              (int)MER_EPI_SPLIT_BF16, (int)MER_EPI_OUT_F16);
  MER_REQUIRE(model->gn_g && model->gn_b, "mer_hubert_conv0: GroupNorm affine missing");
  const long long need = mer_hubert_conv0_workspace_bytes(batch);
  MER_REQUIRE(workspace && workspace_bytes >= need && reinterpret_cast<uintptr_t>(workspace) % 16 == 0,
              "mer_hubert_conv0: workspace %lld B < required %lld B, or not 16-byte aligned", workspace_bytes, need);
  return mer_hubert_conv0_launch(wave, ld_wave, batch, n_samples, model->conv0_w, model->gn_g, model->gn_b,
                                 static_cast<double*>(workspace), static_cast<float*>(out), out_bstride,
                                 out_format == MER_EPI_OUT_F16 ? 2 : 1, s, frames);
}

// the moments ([batch, 128] doubles, MOM_LD used) and then the coefficients ([batch, 512] float2)
extern "C" long long mer_hubert_conv0_workspace_bytes(int batch) {
  return batch > 0 ? (long long)batch * (128 * sizeof(double) + C0 * sizeof(float2)) : 0;
}
