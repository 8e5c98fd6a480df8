// helpers.cu — small HBM-bound kernels around the encoders: ViT frame preprocessing + patch
// gather, CLS rows, and the segment reduce used by every readout.
#include <math.h>

#include <vector>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

// One thread = one 16-pixel row of one 16x16 patch, all 3 channels: reads 48 contiguous bytes of
// the uint8 BGR HWC frame, writes three 64-byte runs of the patch-major GEMM operand
//   A[(n, py, px), c*256 + i*16 + j] = ((frame[n, py*16+i, px*16+j, 2-c] * (1/255)) - 0.5) / 0.5
// (BGR->RGB of extract_vision_huggingface.py:29-31, then HF ViTImageProcessor rescale+normalize),
// rounded to tf32 because its only consumer is the patch-embedding GEMM.
// Algorithmic traffic per frame: 150,528 B in + 602,112 B out.
__global__ void __launch_bounds__(256)
vit_patchify_kernel(const uint8_t* __restrict__ frames, float* __restrict__ a, long long total) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int i = idx & 15;               // row inside the patch
  const long long patch = idx >> 4;     // (n*14 + py)*14 + px
  const int px = patch % 14;
  const long long t = patch / 14;
  const int py = t % 14;
  const long long n = t / 14;
  const uint8_t* src = frames + ((n * 224 + (py * 16 + i)) * 224 + px * 16) * 3;
  uint4 raw[3];
  raw[0] = __ldg(reinterpret_cast<const uint4*>(src));
  raw[1] = __ldg(reinterpret_cast<const uint4*>(src) + 1);
  raw[2] = __ldg(reinterpret_cast<const uint4*>(src) + 2);
  const uint8_t* b = reinterpret_cast<const uint8_t*>(raw);
  float* dst = a + patch * 768 + i * 16;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float p = (float)b[j * 3 + (2 - c)];
      v[j] = round_tf32((p * 0.00392156862745098f - 0.5f) / 0.5f);
    }
    float4* d4 = reinterpret_cast<float4*>(dst + c * 256);
#pragma unroll
    for (int q = 0; q < 4; ++q) d4[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  }
}

// One pass of Pillow's 8-bit bilinear resampling (src/libImaging/Resample.c, ImagingResampleHorizontal_8bpc
// / Vertical_8bpc; reached through HF ViTImageProcessor.resize from extract_vision_huggingface.py:137-138)
// over uint8 HWC frames: out = clip8((2^21 + sum_k in[lo + k] * kk[k]) >> 22) along one axis.
// One thread = one output pixel (3 channels).  in: [n, H, W, 3]; AXIS 0: rows H -> OUT; AXIS 1: columns W -> OUT.
template <int AXIS>
__global__ void __launch_bounds__(256)
resize_pass_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, long long total, int H, int W,
                   int OUT, const int* __restrict__ lo, const int* __restrict__ cnt,
                   const int* __restrict__ kk, int ksize) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int oh = AXIS == 0 ? OUT : H, ow = AXIS == 1 ? OUT : W;
  const int x = (int)(idx % ow);
  const int y = (int)((idx / ow) % oh);
  const long long n = idx / ((long long)ow * oh);
  const int o = AXIS == 0 ? y : x;
  const int first = __ldg(lo + o), m = __ldg(cnt + o);
  int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
  for (int k = 0; k < m; ++k) {
    const int w = __ldg(kk + o * ksize + k);
    const int sy = AXIS == 0 ? first + k : y, sx = AXIS == 1 ? first + k : x;
    const uint8_t* p = in + ((n * H + sy) * W + sx) * 3;
    a0 += (int)p[0] * w;
    a1 += (int)p[1] * w;
    a2 += (int)p[2] * w;
  }
  uint8_t* d = out + idx * 3;
  d[0] = (uint8_t)min(max(a0 >> 22, 0), 255);
  d[1] = (uint8_t)min(max(a1 >> 22, 0), 255);
  d[2] = (uint8_t)min(max(a2 >> 22, 0), 255);
}

// Generic patch gather for the CLIP vision towers: uint8 BGR HWC frames [n, H, W, 3] (a size x size window
// at (y0, x0): the processor's center crop) -> A[(n, py, px), c*p*p + i*p + j] = (frame[..., 2-c] / 255 -
// mean[c]) / std[c], tf32-rounded; columns 3*p*p .. kpad-1 are zero (the GEMM's K is a multiple of 32).
// One thread per output element; consecutive threads write consecutive columns.
__global__ void __launch_bounds__(256)
patchify_generic_kernel(const uint8_t* __restrict__ frames, int H, int W, int y0, int x0, int size, int p,
                        int kpad, float m0, float m1, float m2, float s0, float s1, float s2,
                        float* __restrict__ a, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int k = (int)(idx % kpad);
  const long long patch = idx / kpad;
  const int g = size / p;
  const int px = (int)(patch % g);
  const int py = (int)((patch / g) % g);
  const long long n = patch / ((long long)g * g);
  float v = 0.f;
  if (k < 3 * p * p) {
    const int c = k / (p * p), r = k - c * p * p, i = r / p, j = r - i * p;
    const float pix = (float)frames[((n * H + (y0 + py * p + i)) * W + (x0 + px * p + j)) * 3 + (2 - c)];
    const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), std = c == 0 ? s0 : (c == 1 ? s1 : s2);
    v = round_tf32((pix * 0.00392156862745098f - mean) / std);
  }
  a[idx] = v;
}

// x[n * tokens, :] = row  (class-token row: class embedding + position embedding 0)
__global__ void cls_rows_generic_kernel(const float* __restrict__ row, float* __restrict__ x, int tokens, int dim) {
  float* dst = x + (long long)blockIdx.x * tokens * dim;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) dst[i] = __ldg(row + i);
}

// out[i, :] = in[(first + i * step), :]
__global__ void gather_rows_kernel(const float* __restrict__ in, long long first, long long step, int dim,
                                   float* __restrict__ out) {
  const float* src = in + (first + (long long)blockIdx.x * step) * dim;
  float* dst = out + (long long)blockIdx.x * dim;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) dst[i] = src[i];
}

// x[n, 0, :] = cls_token + position_embeddings[0]  (HF ViTEmbeddings, modeling_vit.py:117-124)
__global__ void vit_cls_rows_kernel(const float* __restrict__ cls_pos0, float* __restrict__ x,
                                    int n_frames) {
  const int n = blockIdx.x;
  if (n >= n_frames) return;
  float4* dst = reinterpret_cast<float4*>(x + (long long)n * 197 * 768);
  dst[threadIdx.x] = __ldg(reinterpret_cast<const float4*>(cls_pos0) + threadIdx.x);
}

// out[s, :] = sum|mean over rows [offsets[s], offsets[s+1]) of in[:, dim].  One block per
// (segment, 512-column slab); 4 row-groups of 128 threads each stride over the rows with float4
// loads and are combined through shared memory.  Algorithmic traffic: rows*dim*4 B in.
__global__ void __launch_bounds__(512)
segment_reduce_kernel(const float* __restrict__ in, const int* __restrict__ begins,
                      const int* __restrict__ ends, int dim, int mode, float* __restrict__ out) {
  __shared__ float4 part[4][128];
  const int s = blockIdx.x;
  const int col4 = blockIdx.y * 128 + (threadIdx.x & 127);  // float4 column
  const int grp = threadIdx.x >> 7;
  const int r0 = begins[s], r1 = max(ends[s], begins[s]);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (col4 * 4 < dim) {
    for (int r = r0 + grp; r < r1; r += 4) {
      const float4 v = *reinterpret_cast<const float4*>(in + (long long)r * dim + col4 * 4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  part[grp][threadIdx.x & 127] = acc;
  __syncthreads();
  if (grp == 0 && col4 * 4 < dim) {
    float4 a = part[0][threadIdx.x], b = part[1][threadIdx.x], c = part[2][threadIdx.x],
           d = part[3][threadIdx.x];
    float4 r;
    r.x = (a.x + b.x) + (c.x + d.x);
    r.y = (a.y + b.y) + (c.y + d.y);
    r.z = (a.z + b.z) + (c.z + d.z);
    r.w = (a.w + b.w) + (c.w + d.w);
    if (mode == MER_SEG_MEAN && r1 > r0) {
      const float inv = 1.0f / (float)(r1 - r0);
      r.x *= inv; r.y *= inv; r.z *= inv; r.w *= inv;
    }
    *reinterpret_cast<float4*>(out + (long long)s * dim + col4 * 4) = r;
  }
}

// BERT/RoBERTa embeddings (HF modeling_bert.py BertEmbeddings / modeling_roberta.py:56-122):
// (word[id] + token_type[0]) + position[pos] -> LayerNorm -> x (fp32) and its split-bf16 copy.
// One warp per token; width 128 * VEC (VEC 6: the base models, VEC 8: the -large ones, VEC 2: LERT-small's hidden 256,
// VEC 1: ELECTRA-small's factorised 128-wide embedding).
template <int VEC>
__global__ void __launch_bounds__(256)
bert_embed_ln_kernel(const int* __restrict__ ids, const int* __restrict__ pos_ids,
                     const float* __restrict__ word, const float* __restrict__ pos,
                     const float* __restrict__ type0, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, int tokens, float* __restrict__ out,
                     void* __restrict__ out_split) {
  constexpr int DIM = 128 * VEC;
  const int lane = threadIdx.x & 31;
  const int tok = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (tok >= tokens) return;
  const float4* w = reinterpret_cast<const float4*>(word + (long long)ids[tok] * DIM);
  const float4* p = reinterpret_cast<const float4*>(pos + (long long)pos_ids[tok] * DIM);
  const float4* ty = reinterpret_cast<const float4*>(type0);
  float4 v[VEC];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const float4 a = __ldg(w + lane + 32 * i), b = __ldg(ty + lane + 32 * i), c = __ldg(p + lane + 32 * i);
    v[i].x = (a.x + b.x) + c.x; v[i].y = (a.y + b.y) + c.y;
    v[i].z = (a.z + b.z) + c.z; v[i].w = (a.w + b.w) + c.w;
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
  float4* o = reinterpret_cast<float4*>(out + (long long)tok * DIM);
  float* os = out_split ? reinterpret_cast<float*>(out_split) + (long long)tok * DIM : nullptr;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i);
    const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + lane + 32 * i);
    float4 r;
    r.x = v[i].x * rstd * g.x + b.x; r.y = v[i].y * rstd * g.y + b.y;
    r.z = v[i].z * rstd * g.z + b.z; r.w = v[i].w * rstd * g.w + b.w;
    if (os) store_split4(os, 4 * (lane + 32 * i), r);
    o[lane + 32 * i] = r;
  }
}

__global__ void iota_offsets_kernel(int* offsets, int n_seg, int step) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= n_seg) offsets[i] = i * step;
}

}  // namespace

int mer_vit_patchify_launch(const uint8_t* frames_bgr, int n_frames, float* a_patches,
                            cudaStream_t stream) {
  const long long total = (long long)n_frames * 196 * 16;
  if (total <= 0) return 0;
  vit_patchify_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(frames_bgr, a_patches,
                                                                           total);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_vit_cls_rows_launch(const float* cls_pos0, float* x, int n_frames, cudaStream_t stream) {
  if (n_frames <= 0) return 0;
  vit_cls_rows_kernel<<<n_frames, 192, 0, stream>>>(cls_pos0, x, n_frames);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_patchify_generic_launch(const uint8_t* frames, int n, int H, int W, int y0, int x0, int size, int patch,
                                int kpad, const float mean[3], const float std[3], float* a, cudaStream_t stream) {
  MER_REQUIRE(size % patch == 0 && kpad >= 3 * patch * patch && y0 >= 0 && x0 >= 0 && y0 + size <= H && x0 + size <= W,
              "mer_patchify_generic: bad geometry");
  const long long g = size / patch;
  const long long total = (long long)n * g * g * kpad;
  patchify_generic_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(
      frames, H, W, y0, x0, size, patch, kpad, mean[0], mean[1], mean[2], std[0], std[1], std[2], a, total);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_cls_rows_generic_launch(const float* row, float* x, int n_frames, int tokens, int dim, cudaStream_t stream) {
  if (n_frames <= 0) return 0;
  cls_rows_generic_kernel<<<n_frames, 256, 0, stream>>>(row, x, tokens, dim);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_gather_rows_launch(const float* in, long long first, long long step, int n, int dim, float* out,
                           cudaStream_t stream) {
  if (n <= 0) return 0;
  gather_rows_kernel<<<n, 256, 0, stream>>>(in, first, step, dim, out);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_segment_reduce_launch(const float* in, const int* begins, const int* ends, int n_seg,
                              int dim, int mode, float* out, cudaStream_t stream) {
  MER_REQUIRE(in && begins && ends && out, "mer_segment_reduce: null operand");
  MER_REQUIRE(dim > 0 && dim % 4 == 0, "mer_segment_reduce: dim %d must be a multiple of 4", dim);
  if (n_seg <= 0) return 0;
  dim3 grid(n_seg, (dim + 511) / 512);
  segment_reduce_kernel<<<grid, 512, 0, stream>>>(in, begins, ends, dim, mode, out);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_bert_embed_launch(const int* ids, const int* pos_ids, const float* word, const float* pos,
                          const float* type0, const float* gamma, const float* beta, float eps,
                          int tokens, float* out, void* out_split, cudaStream_t stream, int dim) {
  if (tokens <= 0) return 0;
  MER_REQUIRE(dim == 768 || dim == 1024 || dim == 128 || dim == 256,
              "mer_bert_embed: hidden size %d (768 or 1024; also 128 and 256)", dim);
#define MER_EMBED_LAUNCH(VEC)                                                                                       \
  bert_embed_ln_kernel<VEC><<<(tokens + 7) / 8, 256, 0, stream>>>(ids, pos_ids, word, pos, type0, gamma, beta, eps, \
                                                                  tokens, out, out_split)
  if (dim == 1024) MER_EMBED_LAUNCH(8);
  else if (dim == 768) MER_EMBED_LAUNCH(6);
  else if (dim == 256) MER_EMBED_LAUNCH(2);
  else MER_EMBED_LAUNCH(1);
#undef MER_EMBED_LAUNCH
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_iota_offsets_launch(int* offsets, int n_seg, int step, cudaStream_t stream) {
  iota_offsets_kernel<<<(n_seg + 256) / 256, 256, 0, stream>>>(offsets, n_seg, step);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

extern "C" int mer_segment_reduce(const float* in, const int32_t* begins, const int32_t* ends,
                                  int n_seg, int dim, int mode, float* out, void* stream) {
  return mer_segment_reduce_launch(in, begins, ends, n_seg, dim, mode, out,
                                   static_cast<cudaStream_t>(stream));
}

// ---- Pillow bilinear resize (uint8) ----------------------------------------------------------------
namespace {
struct ResizeTable { int in, out, filter, ksize; int* d_lo; int* d_cnt; int* d_kk; };
std::vector<ResizeTable> g_resize_tables;  // per process (= per device: one process per GPU)

// Pillow's filters (Resample.c): bilinear (support 1) and bicubic with a = -0.5 (support 2)
double pil_filter(int filter, double x) {
  if (filter == 0) return x < 1.0 ? 1.0 - x : 0.0;
  const double a = -0.5;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

// Pillow precompute_coeffs + normalize_coeffs_8bpc, in double as Pillow does.  filter: 0 bilinear, 1 bicubic
int resize_table(int in_size, int out_size, int filter, const ResizeTable** res, cudaStream_t stream) {
  for (auto& t : g_resize_tables)
    if (t.in == in_size && t.out == out_size && t.filter == filter) { *res = &t; return 0; }
  const double scale = (double)in_size / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = (filter == 0 ? 1.0 : 2.0) * filterscale;
  const int ksize = (int)ceil(support) * 2 + 1;
  std::vector<int> lo(out_size), cnt(out_size), kk((size_t)out_size * ksize, 0);
  std::vector<double> w(ksize);
  const double ss = 1.0 / filterscale;
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    int a = (int)(center - support + 0.5);
    if (a < 0) a = 0;
    int b = (int)(center + support + 0.5);
    if (b > in_size) b = in_size;
    const int n = b - a;
    double tot = 0.0;
    for (int x = 0; x < n; ++x) {
      double v = (x + a - center + 0.5) * ss;
      if (v < 0.0) v = -v;
      w[x] = pil_filter(filter, v);
      tot += w[x];
    }
    for (int x = 0; x < n; ++x) {
      const double k = tot != 0.0 ? w[x] / tot : w[x];
      kk[(size_t)xx * ksize + x] = (int)(k * (double)(1 << 22) + (k < 0 ? -0.5 : 0.5));
    }
    lo[xx] = a;
    cnt[xx] = n;
  }
  ResizeTable t{in_size, out_size, filter, ksize, nullptr, nullptr, nullptr};
  MER_CUDA_CHECK(cudaMalloc(&t.d_lo, out_size * sizeof(int)));
  MER_CUDA_CHECK(cudaMalloc(&t.d_cnt, out_size * sizeof(int)));
  MER_CUDA_CHECK(cudaMalloc(&t.d_kk, kk.size() * sizeof(int)));
  // pageable-host copies are staged before the call returns, so the vectors may go out of scope
  MER_CUDA_CHECK(cudaMemcpyAsync(t.d_lo, lo.data(), out_size * sizeof(int), cudaMemcpyHostToDevice, stream));
  MER_CUDA_CHECK(cudaMemcpyAsync(t.d_cnt, cnt.data(), out_size * sizeof(int), cudaMemcpyHostToDevice, stream));
  MER_CUDA_CHECK(cudaMemcpyAsync(t.d_kk, kk.data(), kk.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
  MER_CUDA_CHECK(cudaStreamSynchronize(stream));
  g_resize_tables.push_back(t);
  *res = &g_resize_tables.back();
  return 0;
}
}  // namespace

extern "C" long long mer_resize_workspace_bytes(int n, int H, int W, int OH, int OW) {
  (void)OH;
  return (H != 0 && W != OW) ? (long long)n * H * OW * 3 : 0;  // the horizontally resampled frames
}

extern "C" int mer_resize_u8(const uint8_t* in, int n, int H, int W, uint8_t* out, int OH, int OW, int filter,
                             void* workspace, void* stream_);

extern "C" int mer_resize_bilinear_u8(const uint8_t* in, int n, int H, int W, uint8_t* out, int OH, int OW,
                                      void* workspace, void* stream_) {
  return mer_resize_u8(in, n, H, W, out, OH, OW, 0, workspace, stream_);
}

extern "C" int mer_resize_u8(const uint8_t* in, int n, int H, int W, uint8_t* out, int OH, int OW, int filter,
                             void* workspace, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(in && out && n > 0 && H > 0 && W > 0 && OH > 0 && OW > 0 && (filter == 0 || filter == 1),
              "mer_resize_u8: bad arguments");
  const bool horiz = W != OW, vert = H != OH;
  if (!horiz && !vert) {
    MER_CUDA_CHECK(cudaMemcpyAsync(out, in, (size_t)n * H * W * 3, cudaMemcpyDeviceToDevice, stream));
    return 0;
  }
  MER_REQUIRE(!(horiz && vert) || workspace, "mer_resize_u8: workspace needed for a two-pass resize");
  const uint8_t* src = in;
  if (horiz) {
    const ResizeTable* t;
    if (int rc = resize_table(W, OW, filter, &t, stream)) return rc;
    uint8_t* dst = vert ? static_cast<uint8_t*>(workspace) : out;
    const long long total = (long long)n * H * OW;
    resize_pass_kernel<1><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(src, dst, total, H, W, OW, t->d_lo,
                                                                               t->d_cnt, t->d_kk, t->ksize);
    MER_CUDA_CHECK(cudaGetLastError());
    mer_count_launches(1);
    src = dst;
  }
  if (vert) {
    const ResizeTable* t;
    if (int rc = resize_table(H, OH, filter, &t, stream)) return rc;
    const long long total = (long long)n * OH * OW;
    resize_pass_kernel<0><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(src, out, total, H, OW, OH, t->d_lo,
                                                                               t->d_cnt, t->d_kk, t->ksize);
    MER_CUDA_CHECK(cudaGetLastError());
    mer_count_launches(1);
  }
  return 0;
}

// ---- cv2.resize(..., INTER_LINEAR) on uint8 HWC frames, bit-exact (OpenCV imgproc/src/resize.cpp: 11-bit fixed-point
// coefficients; the x fraction is reset at the borders, the y rows are only clamped; vertical pass
// ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2 >> 2; an exact 2x downscale is the 2 x 2 area average).
// The EmoNet extractor's DataAugmentor resizes faces this way (emonet/data_augmentation.py:77). ----
namespace {
__device__ __forceinline__ void cv_coeff(int d, double scale, int& s, int& a0, int& a1) {
  float f = (float)__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);  // two roundings, as the host code (no FMA)
  s = (int)floorf(f);
  f -= (float)s;
  a1 = __float2int_rn(f * 2048.f);
  a0 = __float2int_rn((1.f - f) * 2048.f);
}

__global__ void __launch_bounds__(256)
resize_cv2_linear_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, long long total, int H, int W, int OH,
                         int OW, double sy_scale, double sx_scale) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ox = (int)(idx % OW), oy = (int)((idx / OW) % OH);
  const long long n = idx / ((long long)OW * OH);
  const uint8_t* img = in + n * H * W * 3;
  uint8_t* o = out + idx * 3;
  if (H == 2 * OH && W == 2 * OW) {
    const uint8_t* p = img + ((long long)(2 * oy) * W + 2 * ox) * 3;
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)((p[c] + p[3 + c] + p[W * 3 + c] + p[W * 3 + 3 + c] + 2) >> 2);
    return;
  }
  int sx, ax0, ax1, sy, ay0, ay1;
  cv_coeff(ox, sx_scale, sx, ax0, ax1);
  if (sx < 0) { sx = 0; ax0 = 2048; ax1 = 0; }
  if (sx >= W - 1) { sx = W - 1; ax0 = 2048; ax1 = 0; }
  cv_coeff(oy, sy_scale, sy, ay0, ay1);
  const int y0 = min(max(sy, 0), H - 1), y1 = min(max(sy + 1, 0), H - 1), x1 = min(sx + 1, W - 1);
  const uint8_t* r0 = img + (long long)y0 * W * 3;
  const uint8_t* r1 = img + (long long)y1 * W * 3;
  for (int c = 0; c < 3; ++c) {
    const int h0 = r0[sx * 3 + c] * ax0 + r0[x1 * 3 + c] * ax1;
    const int h1 = r1[sx * 3 + c] * ax0 + r1[x1 * 3 + c] * ax1;
    const int v = (((ay0 * (h0 >> 4)) >> 16) + ((ay1 * (h1 >> 4)) >> 16) + 2) >> 2;
    o[c] = (uint8_t)min(max(v, 0), 255);
  }
}
}  // namespace

extern "C" int mer_resize_cv2_linear_u8(const uint8_t* in, int n, int H, int W, uint8_t* out, int OH, int OW,
                                        void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(in && out && in != out && n > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "mer_resize_cv2_linear_u8: bad arguments");
  const long long total = (long long)n * OH * OW;
  resize_cv2_linear_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, out, total, H, W, OH, OW,
                                                                                (double)H / OH, (double)W / OW);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

// ---- VideoMAE tubelet patches (HF VideoMAEPatchEmbeddings: Conv3d(3, hidden, (2, 16, 16), stride = kernel) on
// [B, C, 16, 224, 224]): uint8 BGR frames [B * 16, 224, 224, 3] -> TF32-rounded fp32 rows [B * 1568, 1536], row =
// (tubelet, patch row, patch column), K = (channel, frame in tubelet, dy, dx) = the flattened conv kernel, values
// (pix / 255 - mean[c]) / std[c] in RGB order (VideoMAEImageProcessor's rescale + normalise). ----
namespace {
__global__ void __launch_bounds__(256)
videomae_patchify_kernel(const uint8_t* __restrict__ frames, float* __restrict__ out, long long total, float m0, float m1,
                         float m2, float s0, float s1, float s2) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int k = (int)(idx % 1536);
  const long long row = idx / 1536;
  const int token = (int)(row % 1568);
  const long long b = row / 1568;
  const int c = k >> 9, dt = (k >> 8) & 1, dy = (k >> 4) & 15, dx = k & 15;
  const int tt = token / 196, py = (token % 196) / 14, px = token % 14;
  const long long frame = b * 16 + tt * 2 + dt;
  const float pix = (float)frames[((frame * 224 + py * 16 + dy) * 224 + px * 16 + dx) * 3 + (2 - c)];
  const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
  out[idx] = round_tf32((pix * 0.00392156862745098f - mean) / sd);
}
}  // namespace

extern "C" int mer_videomae_patchify(const uint8_t* frames_bgr, int n_clips, const float* mean, const float* std,
                                     float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(frames_bgr && mean && std && out && n_clips > 0, "mer_videomae_patchify: bad arguments");
  const long long total = (long long)n_clips * 1568 * 1536;
  videomae_patchify_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(frames_bgr, out, total, mean[0], mean[1],
                                                                                mean[2], std[0], std[1], std[2]);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

// ---- SwiGLU gate of HF Dinov2SwiGLUFFN (dinov2-giant): out[r, j] = silu(in[r, j]) * in[r, H + j] for j < H,
// in [rows, 2 H] = weights_in(x); 4 columns per thread, optionally TF32-rounded (operand of weights_out). ----
namespace {
__global__ void __launch_bounds__(256)
swiglu_kernel(const float4* __restrict__ in, float4* __restrict__ out, long long total4, int h4, int round_out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total4) return;
  const long long r = idx / h4;
  const int j = (int)(idx % h4);
  const float4 a = __ldg(in + r * 2 * h4 + j), b = __ldg(in + r * 2 * h4 + h4 + j);
  float4 o;
  o.x = a.x / (1.0f + expf(-a.x)) * b.x;
  o.y = a.y / (1.0f + expf(-a.y)) * b.y;
  o.z = a.z / (1.0f + expf(-a.z)) * b.z;
  o.w = a.w / (1.0f + expf(-a.w)) * b.w;
  if (round_out) o = make_float4(mer::round_tf32(o.x), mer::round_tf32(o.y), mer::round_tf32(o.z), mer::round_tf32(o.w));
  out[idx] = o;
}
}  // namespace

extern "C" int mer_swiglu(const float* in, float* out, long long rows, int hidden, int round_tf32_out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(in && out && in != out && rows > 0 && hidden > 0 && hidden % 4 == 0, "mer_swiglu: bad arguments");
  const long long total4 = rows * (hidden / 4);
  swiglu_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(in),
                                                                      reinterpret_cast<float4*>(out), total4, hidden / 4,
                                                                      round_tf32_out);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}
