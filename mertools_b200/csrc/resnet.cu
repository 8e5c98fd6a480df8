// resnet.cu — the convolutional extractors: ResNet-18 frame encoder of the reference's ImageNet CNN extractor
// (MERBench/feature_extraction/visual/extract_imagenet_embedding.py:47-55: torchvision resnet18 without its
// fc layer on Resize(224) / ToTensor / Normalize(ImageNet) frames -> one 512-vector per frame).
//
// Every convolution (BatchNorm folded into weight and bias at load time) is an im2col gather into an fp16
// operand followed by the shared wgmma GEMM (MER_GEMM_F16) with its epilogue doing bias (+ identity)
// + ReLU; activations stay NHWC fp32 between layers (the GEMM's residual input is fp32).  64-channel layers
// are stored with 128 channels (upper half zero) because the GEMM's narrowest column block is 128; the gather
// reads only the real channels, so K is not inflated.  Max-pool and the im2col gathers are plain coalesced
// kernels (HBM-bound); the global average pool is the shared segment reduce.
// Per frame: 1.82 GFLOP algorithmic (2.4 executed with the 64 -> 128 column padding).
#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

// conv1 gather: uint8 BGR frames [n, 224, 224, 3] -> rows (n, oy, ox) of K = 7*7*3 (ky, kx, c) operand values
// ((pix * scale - mean[c]) / std[c], RGB order: ToTensor [* 255] + Normalize), zero outside the image and for
// k >= 147.  SPLIT = false: fp16, kpad 192; SPLIT = true: bf16 hi | lo groups (MER_GEMM_BF16X3), kpad 160.
template <bool SPLIT>
__global__ void __launch_bounds__(256)
im2col_stem_kernel(const uint8_t* __restrict__ frames, int H, int W, int OH, int OW, int kpad, float scale, float m0,
                   float m1, float m2, float s0, float s1, float s2, uint16_t* __restrict__ out, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int k = (int)(idx % kpad);
  const long long row = idx / kpad;
  const int ox = (int)(row % OW), oy = (int)((row / OW) % OH);
  const long long n = row / ((long long)OW * OH);
  float v = 0.f;
  if (k < 147) {
    const int c = k % 3, kx = (k / 3) % 7, ky = k / 21;
    const int iy = oy * 2 - 3 + ky, ix = ox * 2 - 3 + kx;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
      const float pix = (float)frames[((n * H + iy) * W + ix) * 3 + (2 - c)];
      const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
      v = (pix * scale - mean) / sd;
    }
  }
  if (SPLIT) {
    uint16_t* grp = out + row * (long long)kpad * 2 + (k >> 5) * 64 + (k & 31);
    const float hi = bf16_round(v);
    grp[0] = (uint16_t)(__float_as_uint(hi) >> 16);
    grp[32] = (uint16_t)(pack_bf16x2(v - hi, 0.f) & 0xffffu);
  } else {
    out[idx] = (uint16_t)(pack_f16x2(v, 0.f) & 0xffffu);
  }
}

// generic gather: NHWC fp32 activations [n, H, W, cs] (first C channels real) -> operand rows (n, oy, ox) of
// K = k*k*C values in (ky, kx, c) order; one thread = 8 consecutive channels.  SPLIT = false: fp16 (16 bytes
// out, MER_GEMM_F16); SPLIT = true: bf16 hi | lo in the 128-byte groups of MER_GEMM_BF16X3 (two 16-byte stores:
// 8 consecutive K indices never straddle a 32-value group).
template <bool SPLIT>
__global__ void __launch_bounds__(256)
im2col_kernel(const float* __restrict__ x, int H, int W, int cs, int C, int ksz, int stride, int pad, int OH, int OW,
              uint4* __restrict__ out, long long total8) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total8) return;
  const int c8 = C / 8;
  const int kc = ksz * ksz * c8;
  const int q = (int)(idx % kc);
  const long long row = idx / kc;
  const int cg = q % c8, kx = (q / c8) % ksz, ky = q / (c8 * ksz);
  const int ox = (int)(row % OW), oy = (int)((row / OW) % OH);
  const long long n = row / ((long long)OW * OH);
  const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
  if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
    const float4* src = reinterpret_cast<const float4*>(x + ((n * H + iy) * W + ix) * (long long)cs + cg * 8);
    a = __ldg(src);
    b = __ldg(src + 1);
  }
  if (SPLIT) {
    const int k = q * 8;  // K index of the first of the 8 values
    uint4* grp = out + (row * kc + (k >> 5) * 4) * 2 + ((k & 31) >> 3);  // 16-byte slot of the hi half
    const float h0 = bf16_round(a.x), h1 = bf16_round(a.y), h2 = bf16_round(a.z), h3 = bf16_round(a.w);
    const float h4 = bf16_round(b.x), h5 = bf16_round(b.y), h6 = bf16_round(b.z), h7 = bf16_round(b.w);
    grp[0] = make_uint4(pack_bf16x2(h0, h1), pack_bf16x2(h2, h3), pack_bf16x2(h4, h5), pack_bf16x2(h6, h7));
    grp[4] = make_uint4(pack_bf16x2(a.x - h0, a.y - h1), pack_bf16x2(a.z - h2, a.w - h3),
                        pack_bf16x2(b.x - h4, b.y - h5), pack_bf16x2(b.z - h6, b.w - h7));
  } else {
    out[idx] = make_uint4(pack_f16x2(a.x, a.y), pack_f16x2(a.z, a.w), pack_f16x2(b.x, b.y), pack_f16x2(b.z, b.w));
  }
}

// MaxPool2d(3, stride 2, padding pad) on NHWC fp32, 4 channels per thread; windows are clipped to the image
// (padding 1: torchvision ResNet; padding 0 with ceil_mode: the caffe-style FER+ models)
__global__ void __launch_bounds__(256)
maxpool3x3s2_kernel(const float4* __restrict__ x, int H, int W, int c4, int OH, int OW, int pad, float4* __restrict__ y,
                    long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = (int)(idx % c4);
  const long long pos = idx / c4;
  const int ox = (int)(pos % OW), oy = (int)((pos / OW) % OH);
  const long long n = pos / ((long long)OW * OH);
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = oy * 2 - pad + ky;
    if (iy < 0 || iy >= H) continue;
    for (int kx = 0; kx < 3; ++kx) {
      const int ix = ox * 2 - pad + kx;
      if (ix < 0 || ix >= W) continue;
      const float4 v = __ldg(x + ((n * H + iy) * W + ix) * (long long)c4 + c);
      m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
    }
  }
  y[idx] = m;
}

// VGGish conv1 gather: fp32 log-mel examples [n, H, W] (one channel) -> split-bf16 rows (n, y, x) of K = 9 taps
// (ky, kx) zero-padded to one 32-value group = 128 bytes [32 hi | 32 lo]; one thread = one 16-byte slot
// (slots 0..3: hi of taps 8 s .. 8 s + 7, slots 4..7: the lo halves).
__global__ void __launch_bounds__(256)
im2col_1ch_kernel(const float* __restrict__ x, int H, int W, uint4* __restrict__ out, long long total_slots) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total_slots) return;
  const int slot = (int)(idx & 7), ks = (slot & 3) * 8;
  uint4 o = make_uint4(0u, 0u, 0u, 0u);
  if (ks < 9) {
    const long long row = idx >> 3;
    const int px = (int)(row % W), py = (int)((row / W) % H);
    const float* img = x + (row / ((long long)W * H)) * H * W;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = ks + j, iy = py - 1 + k / 3, ix = px - 1 + k % 3;
      const float val = (k < 9 && iy >= 0 && iy < H && ix >= 0 && ix < W) ? __ldg(img + iy * W + ix) : 0.f;
      const float hi = bf16_round(val);
      v[j] = slot < 4 ? hi : val - hi;
    }
    o = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
  }
  out[idx] = o;
}

// max_pool2d 2x2 / stride 2 on NHWC fp32 (even H and W: TF 'SAME' == 'VALID'), 4 channels per thread
__global__ void __launch_bounds__(256)
maxpool2x2_kernel(const float4* __restrict__ x, int H, int W, int c4, float4* __restrict__ y, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int OW = W / 2, OH = H / 2;
  const int c = (int)(idx % c4);
  const long long pos = idx / c4;
  const int ox = (int)(pos % OW), oy = (int)((pos / OW) % OH);
  const long long n = pos / ((long long)OW * OH);
  const float4* p = x + ((n * H + 2 * oy) * W + 2 * ox) * (long long)c4 + c;
  const float4 a = __ldg(p), b = __ldg(p + c4), d = __ldg(p + (long long)W * c4), e = __ldg(p + (long long)(W + 1) * c4);
  y[idx] = make_float4(fmaxf(fmaxf(a.x, b.x), fmaxf(d.x, e.x)), fmaxf(fmaxf(a.y, b.y), fmaxf(d.y, e.y)),
                       fmaxf(fmaxf(a.z, b.z), fmaxf(d.z, e.z)), fmaxf(fmaxf(a.w, b.w), fmaxf(d.w, e.w)));
}

// squeeze-and-excitation gate of senet50_ferplus_dag: scale[n, c] = sigmoid(up(relu(down(z[n, :])))) with z the
// per-frame channel means; one block per frame, fp32 (2 * C * C/16 MACs per frame)
__global__ void __launch_bounds__(256)
se_mlp_kernel(const float* __restrict__ z, const float* __restrict__ wd, const float* __restrict__ bd,
              const float* __restrict__ wu, const float* __restrict__ bu, int C, int R, float* __restrict__ scale) {
  extern __shared__ float se_sm[];
  float* zs = se_sm;
  float* ds = se_sm + C;
  const long long n = blockIdx.x;
  for (int i = threadIdx.x; i < C; i += blockDim.x) zs[i] = z[n * C + i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < R; j += 8) {
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a = fmaf(__ldg(wd + (long long)j * C + c), zs[c], a);
    a = warp_sum(a);
    if (lane == 0) ds[j] = fmaxf(a + __ldg(bd + j), 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = __ldg(bu + c);
    for (int j = 0; j < R; ++j) a = fmaf(__ldg(wu + (long long)c * R + j), ds[j], a);
    scale[n * C + c] = 1.0f / (1.0f + expf(-a));
  }
}

// out = relu(scale[n, c] * y + res) on NHWC fp32 maps (C == stored channels), 4 channels per thread
__global__ void __launch_bounds__(256)
se_apply_kernel(const float4* __restrict__ y, const float4* __restrict__ res, const float4* __restrict__ scale,
                long long hw_c4, int c4, float4* __restrict__ out, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const float4 sc = __ldg(scale + (idx / hw_c4) * c4 + idx % c4);
  const float4 a = __ldg(y + idx), r = __ldg(res + idx);
  out[idx] = make_float4(fmaxf(fmaf(sc.x, a.x, r.x), 0.f), fmaxf(fmaf(sc.y, a.y, r.y), 0.f),
                         fmaxf(fmaf(sc.z, a.z, r.z), 0.f), fmaxf(fmaf(sc.w, a.w, r.w), 0.f));
}

struct Shape { int H, W, C, Cs; };  // C real channels, Cs stored channels (>= 128)

// mode: MER_GEMM_F16 (fp16 operand, weights fp16) or MER_GEMM_BF16X3 (split-bf16 operand and weights)
int conv(const MerResnetConv& cv, const float* x, Shape in, int n, uint16_t* col, const float* res, bool relu,
         float* y, Shape* out, cudaStream_t st, int mode = MER_GEMM_F16) {
  const int OH = (in.H + 2 * cv.pad - cv.k) / cv.stride + 1, OW = (in.W + 2 * cv.pad - cv.k) / cv.stride + 1;
  const long long rows = (long long)n * OH * OW;
  const int K = cv.k * cv.k * in.C;
  const bool split = mode == MER_GEMM_BF16X3;
  MER_REQUIRE(cv.cin == in.C && cv.kpad == K && K % (split ? 32 : 64) == 0 && in.C % 8 == 0,
              "conv: geometry (cin %d K %d)", cv.cin, K);
  const long long total8 = rows * (K / 8);
  const unsigned blocks = (unsigned)((total8 + 255) / 256);
  if (split)
    im2col_kernel<true><<<blocks, 256, 0, st>>>(x, in.H, in.W, in.Cs, in.C, cv.k, cv.stride, cv.pad, OH, OW,
                                                reinterpret_cast<uint4*>(col), total8);
  else
    im2col_kernel<false><<<blocks, 256, 0, st>>>(x, in.H, in.W, in.Cs, in.C, cv.k, cv.stride, cv.pad, OH, OW,
                                                 reinterpret_cast<uint4*>(col), total8);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  MerGemmDesc g;
  memset(&g, 0, sizeof(g));
  g.A = reinterpret_cast<const float*>(col);
  g.W = static_cast<const float*>(cv.w);
  g.rows_per_batch = (int)rows;
  g.a_rows_dim = (int)rows;
  g.batches = 1;
  g.N = cv.cout_pad;
  g.K_inner = K;
  g.taps = 1;
  g.P = 1;
  g.a_phase_stride = K;
  g.a_row_stride = K;
  g.a_batch_stride = rows * K;
  g.mode = mode;
  g.ep.bias = cv.b;
  g.ep.res = res;
  g.ep.out = y;
  g.ep.ld_out = cv.cout_pad;
  g.ep.ld_res = cv.cout_pad;
  g.ep.flags = relu ? MER_EPI_RELU : 0;
  if (int rc = mer_gemm_launch(&g, st)) return rc;
  *out = Shape{OH, OW, cv.cout, cv.cout_pad};
  return 0;
}

}  // namespace

namespace {
struct ResnetPlan { long long off_a0, off_p, off_q, off_r, off_col, off_cu, total; };
ResnetPlan resnet_plan(int n_frames) {
  const long long n = n_frames;
  auto al = [](long long x) { return (x + 255) & ~255ll; };
  ResnetPlan p;
  long long o = 0;
  p.off_a0 = o;  o += al(n * 112 * 112 * 128 * 4);   // conv1 output (64 real channels stored as 128)
  p.off_p = o;   o += al(n * 56 * 56 * 128 * 4);     // residual stream
  p.off_q = o;   o += al(n * 56 * 56 * 128 * 4);     // block-internal activation
  p.off_r = o;   o += al(n * 28 * 28 * 128 * 4);     // downsample branch (first needed at 28 x 28)
  const long long c1 = n * 112 * 112 * 192 * 2, c2 = n * 56 * 56 * 576 * 2;
  p.off_col = o; o += al(c1 > c2 ? c1 : c2);         // fp16 im2col operand
  p.off_cu = o;  o += al((n + 1) * 4);
  p.total = o;
  return p;
}
}  // namespace

extern "C" {

long long mer_resnet18_workspace_bytes(int n_frames) { return resnet_plan(n_frames).total; }

int mer_resnet18_forward(const MerResnet18Model* m, const uint8_t* frames_bgr, int n_frames, void* workspace,
                         long long workspace_bytes, float* out_feats, void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(m && frames_bgr && workspace && out_feats && n_frames > 0, "mer_resnet18_forward: bad operands");
  const ResnetPlan p = resnet_plan(n_frames);
  MER_REQUIRE(workspace_bytes >= p.total, "mer_resnet18_forward: workspace %lld B < required %lld B", workspace_bytes,
              p.total);
  MER_REQUIRE((long long)n_frames * 112 * 112 < (1ll << 31), "mer_resnet18_forward: too many frames per call");
  const long long n = n_frames;
  char* ws = static_cast<char*>(workspace);
  float* a0 = reinterpret_cast<float*>(ws + p.off_a0);
  float* x = reinterpret_cast<float*>(ws + p.off_p);
  float* t1 = reinterpret_cast<float*>(ws + p.off_q);
  float* t2 = reinterpret_cast<float*>(ws + p.off_r);
  uint16_t* col = reinterpret_cast<uint16_t*>(ws + p.off_col);
  int* offsets = reinterpret_cast<int*>(ws + p.off_cu);

  // stem: conv1 7x7/2 (+BN folded) + ReLU
  {
    const MerResnetConv& cv = m->convs[0];
    MER_REQUIRE(cv.k == 7 && cv.kpad == 192 && cv.cout_pad == 128, "mer_resnet18_forward: conv1 packing");
    const long long rows = n * 112 * 112, total = rows * 192;
    im2col_stem_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
        frames_bgr, 224, 224, 112, 112, 192, 0.00392156862745098f, m->mean[0], m->mean[1], m->mean[2], m->std[0],
        m->std[1], m->std[2], col, total);
    MER_CUDA_CHECK(cudaGetLastError());
    mer_count_launches(1);
    MerGemmDesc g;
    memset(&g, 0, sizeof(g));
    g.A = reinterpret_cast<const float*>(col);
    g.W = static_cast<const float*>(cv.w);
    g.rows_per_batch = (int)rows;
    g.a_rows_dim = (int)rows;
    g.batches = 1;
    g.N = 128;
    g.K_inner = 192;
    g.taps = 1;
    g.P = 1;
    g.a_phase_stride = 192;
    g.a_row_stride = 192;
    g.a_batch_stride = rows * 192;
    g.mode = MER_GEMM_F16;
    g.ep.bias = cv.b;
    g.ep.out = a0;
    g.ep.ld_out = 128;
    g.ep.flags = MER_EPI_RELU;
    if (int rc = mer_gemm_launch(&g, st)) return rc;
  }
  // maxpool 3x3/2 -> x [n,56,56,128]
  {
    const long long total = n * 56 * 56 * 32;
    maxpool3x3s2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float4*>(a0), 112, 112, 32,
                                                                         56, 56, 1, reinterpret_cast<float4*>(x), total);
    MER_CUDA_CHECK(cudaGetLastError());
    mer_count_launches(1);
  }
  // four stages of two BasicBlocks (torchvision resnet.py: conv-bn-relu, conv-bn, (+downsample), add, relu).
  // The block output overwrites the stream buffer: its residual is either the stream itself (read and written
  // by the same epilogue thread) or the downsample branch in t2.
  Shape s{56, 56, 64, 128};
  int ci = 1;
  for (int stage = 0; stage < 4; ++stage) {
    for (int blk = 0; blk < 2; ++blk) {
      const bool down = stage > 0 && blk == 0;
      Shape s1, s2, sd;
      if (int rc = conv(m->convs[ci], x, s, n_frames, col, nullptr, true, t1, &s1, st)) return rc;
      const float* identity = x;
      if (down) {
        if (int rc = conv(m->convs[ci + 2], x, s, n_frames, col, nullptr, false, t2, &sd, st)) return rc;
        identity = t2;
      }
      if (int rc = conv(m->convs[ci + 1], t1, s1, n_frames, col, identity, true, x, &s2, st)) return rc;
      s = s2;
      ci += down ? 3 : 2;
    }
  }
  // global average pool over the 7 x 7 positions
  MER_REQUIRE(s.H == 7 && s.W == 7 && s.C == 512 && s.Cs == 512, "mer_resnet18_forward: unexpected final shape");
  if (int rc = mer_iota_offsets_launch(offsets, n_frames, 49, st)) return rc;
  return mer_segment_reduce_launch(x, offsets, offsets + 1, n_frames, 512, MER_SEG_MEAN, out_feats, st);
}

}  // extern "C"

// ---- VGGish (MERBench/feature_extraction/audio/vggish/vggish_slim.py:37-100): six 3x3 'SAME' convolutions with
// ReLU, four 2x2 max-pools, three fully connected layers with ReLU, on [96, 64] log-mel examples.
// All nine GEMMs run MER_GEMM_BF16X3: nothing normalises between the layers, and an fp32 emulation of fp16
// operands put the embedding 1.1e-3 off the fp32 result (every layer adds 2-5e-4), over the 1e-3 bar; at
// 1.7 GFLOP per 0.96 s example the 3x MMA count is immaterial next to the HuBERT path (14 GFLOP per second). ----
namespace {
struct VggishPlan { long long off_a, off_p, off_col, off_h16, off_f, total; };
VggishPlan vggish_plan(int n_examples) {
  const long long n = n_examples;
  auto al = [](long long x) { return (x + 255) & ~255ll; };
  VggishPlan p;
  long long o = 0;
  p.off_a = o;   o += al(n * 96 * 64 * 128 * 4);      // conv outputs (conv1: 64 real channels stored as 128)
  p.off_p = o;   o += al(n * 48 * 32 * 128 * 4);      // pooled maps / the second buffer of a conv pair
  p.off_col = o; o += al(n * 48 * 32 * 576 * 4);      // split-bf16 im2col operand (largest: conv2; conv1 is 96*64*32)
  p.off_h16 = o; o += al(n * 12288 * 4);              // split-bf16 operand of a fully connected layer
  p.off_f = o;   o += al(n * 4096 * 4);               // fp32 output of fc1_1 / fc1_2
  p.total = o;
  return p;
}

// relu(x W^T + b): x fp32 [rows, K] -> split-bf16 scratch -> MER_GEMM_BF16X3 against split-bf16 weights [N, K]
int fc(const void* w_split, const float* b, const float* x, void* x_split, int rows, int K, int N, float* out,
       cudaStream_t st) {
  if (int rc = mer_split_bf16(x, x_split, rows, K, st)) return rc;
  MerGemmDesc g;
  memset(&g, 0, sizeof(g));
  g.A = static_cast<const float*>(x_split);
  g.W = static_cast<const float*>(w_split);
  g.rows_per_batch = rows;
  g.a_rows_dim = rows;
  g.batches = 1;
  g.N = N;
  g.K_inner = K;
  g.taps = 1;
  g.P = 1;
  g.a_phase_stride = K;
  g.a_row_stride = K;
  g.a_batch_stride = (long long)rows * K;
  g.mode = MER_GEMM_BF16X3;
  g.ep.bias = b;
  g.ep.out = out;
  g.ep.ld_out = N;
  g.ep.flags = MER_EPI_RELU;
  return mer_gemm_launch(&g, st);
}

int pool2(const float* x, Shape* s, int n, float* y, cudaStream_t st) {
  const long long total = (long long)n * (s->H / 2) * (s->W / 2) * (s->Cs / 4);
  maxpool2x2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float4*>(x), s->H, s->W,
                                                                     s->Cs / 4, reinterpret_cast<float4*>(y), total);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  s->H /= 2;
  s->W /= 2;
  return 0;
}
}  // namespace

extern "C" {

long long mer_vggish_workspace_bytes(int n_examples) { return vggish_plan(n_examples).total; }

int mer_vggish_forward(const MerVggishModel* m, const float* examples, int n_examples, void* workspace,
                       long long workspace_bytes, float* out_embeddings, void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(m && examples && workspace && out_embeddings && n_examples > 0, "mer_vggish_forward: bad operands");
  const VggishPlan p = vggish_plan(n_examples);
  MER_REQUIRE(workspace_bytes >= p.total, "mer_vggish_forward: workspace %lld B < required %lld B", workspace_bytes,
              p.total);
  MER_REQUIRE((long long)n_examples * 96 * 64 < (1ll << 31), "mer_vggish_forward: too many examples per call");
  char* ws = static_cast<char*>(workspace);
  float* A = reinterpret_cast<float*>(ws + p.off_a);
  float* P = reinterpret_cast<float*>(ws + p.off_p);
  uint16_t* col = reinterpret_cast<uint16_t*>(ws + p.off_col);
  uint16_t* h16 = reinterpret_cast<uint16_t*>(ws + p.off_h16);
  float* F = reinterpret_cast<float*>(ws + p.off_f);
  const int n = n_examples;

  // conv1 (1 -> 64): 9 taps gathered into one 32-value split group
  {
    const MerResnetConv& cv = m->convs[0];
    MER_REQUIRE(cv.k == 3 && cv.cin == 1 && cv.kpad == 32 && cv.cout == 64 && cv.cout_pad == 128,
                "mer_vggish_forward: conv1 packing");
    const long long rows = (long long)n * 96 * 64, slots = rows * 8;
    im2col_1ch_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(examples, 96, 64, reinterpret_cast<uint4*>(col),
                                                                       slots);
    MER_CUDA_CHECK(cudaGetLastError());
    mer_count_launches(1);
    MerGemmDesc g;
    memset(&g, 0, sizeof(g));
    g.A = reinterpret_cast<const float*>(col);
    g.W = static_cast<const float*>(cv.w);
    g.rows_per_batch = (int)rows;
    g.a_rows_dim = (int)rows;
    g.batches = 1;
    g.N = 128;
    g.K_inner = 32;
    g.taps = 1;
    g.P = 1;
    g.a_phase_stride = 32;
    g.a_row_stride = 32;
    g.a_batch_stride = rows * 32;
    g.mode = MER_GEMM_BF16X3;
    g.ep.bias = cv.b;
    g.ep.out = A;
    g.ep.ld_out = 128;
    g.ep.flags = MER_EPI_RELU;
    if (int rc = mer_gemm_launch(&g, st)) return rc;
  }
  Shape s{96, 64, 64, 128};
  if (int rc = pool2(A, &s, n, P, st)) return rc;  // [48, 32, 64]
  if (int rc = conv(m->convs[1], P, s, n, col, nullptr, true, A, &s, st, MER_GEMM_BF16X3)) return rc;  // conv2 -> 128
  if (int rc = pool2(A, &s, n, P, st)) return rc;  // [24, 16, 128]
  if (int rc = conv(m->convs[2], P, s, n, col, nullptr, true, A, &s, st, MER_GEMM_BF16X3)) return rc;  // conv3_1 -> 256
  if (int rc = conv(m->convs[3], A, s, n, col, nullptr, true, P, &s, st, MER_GEMM_BF16X3)) return rc;  // conv3_2
  if (int rc = pool2(P, &s, n, A, st)) return rc;  // [12, 8, 256]
  if (int rc = conv(m->convs[4], A, s, n, col, nullptr, true, P, &s, st, MER_GEMM_BF16X3)) return rc;  // conv4_1 -> 512
  if (int rc = conv(m->convs[5], P, s, n, col, nullptr, true, A, &s, st, MER_GEMM_BF16X3)) return rc;  // conv4_2
  if (int rc = pool2(A, &s, n, P, st)) return rc;  // [6, 4, 512]
  MER_REQUIRE(s.H == 6 && s.W == 4 && s.C == 512 && s.Cs == 512, "mer_vggish_forward: unexpected final shape");
  // slim.flatten of the NHWC map = the buffer as it lies; fc1_1, fc1_2, fc2 (all with ReLU)
  if (int rc = fc(m->fc_w[0], m->fc_b[0], P, h16, n, 12288, 4096, F, st)) return rc;
  if (int rc = fc(m->fc_w[1], m->fc_b[1], F, h16, n, 4096, 4096, A, st)) return rc;  // A is free again
  return fc(m->fc_w[2], m->fc_b[2], A, h16, n, 4096, 128, out_embeddings, st);
}

}  // extern "C"

// ---- table-driven CNN executor (mer_cnn_forward): the frame-level CNN extractors whose graphs are chains of
// conv (+ folded BN, + residual, + ReLU), max-pool, crops / channel slices, gates (SE, CBAM) and average pools over
// up to eight NHWC fp32 activation buffers.  Users: the FER+ ResNet-50 / SENet-50 (extract_ferplus_embedding.py) and
// MA-Net (extract_manet_embedding.py). ----
namespace {

constexpr int CNN_BUFS = 24;

// dst = src[:, y0:y0+h, x0:x0+w, :]  (NHWC fp32, 4 channels per thread)
__global__ void __launch_bounds__(256)
crop_kernel(const float4* __restrict__ x, int H, int W, int c4, int y0, int x0, int h, int w, float4* __restrict__ y,
            long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = (int)(idx % c4);
  const long long pos = idx / c4;
  const int px = (int)(pos % w), py = (int)((pos / w) % h);
  const long long n = pos / ((long long)w * h);
  y[idx] = __ldg(x + ((n * H + y0 + py) * W + x0 + px) * (long long)c4 + c);
}

// dst[r, d0 + j] = f(src[r, s0 + j]) (+ res[r, r0 + j]) for j < width; pre_relu: f = relu; post_relu: relu of the sum.
// Row strides (stored channels) differ per operand; 4 channels per thread.
__global__ void __launch_bounds__(256)
slice_kernel(const float* __restrict__ src, int s_ld, int s0, const float* __restrict__ res, int r_ld, int r0,
             float* __restrict__ dst, int d_ld, int d0, int w4, int pre_relu, int post_relu, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int j = (int)(idx % w4) * 4;
  const long long r = idx / w4;
  float4 v = __ldg(reinterpret_cast<const float4*>(src + r * s_ld + s0 + j));
  if (pre_relu) v = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
  if (res) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(res + r * r_ld + r0 + j));
    v = make_float4(v.x + q.x, v.y + q.y, v.z + q.z, v.w + q.w);
  }
  if (post_relu) v = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
  *reinterpret_cast<float4*>(dst + r * d_ld + d0 + j) = v;
}

// CBAM (manet/model/attention.py:27-84) + shortcut + ReLU on one frame's small map (hw <= 64 positions), one block
// per frame:  cg = sigmoid(mlp(mean_hw y) + mlp(max_hw y));  y1 = y * cg;  comp = [max_c y1, mean_c y1];
// sg = sigmoid(conv7x7(comp) with the BatchNorm folded);  out = relu(y1 * sg + res).
// w1 [R, C], b1 [R], w2 [C, R], b2 [C]: the shared MLP; ws [2 * 49] (+ bs [1]): the folded spatial conv.
__global__ void __launch_bounds__(256)
cbam_kernel(const float* __restrict__ y, const float* __restrict__ res, const float* __restrict__ w1,
            const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
            const float* __restrict__ wsp, const float* __restrict__ bsp, int H, int W, int C, int R,
            float* __restrict__ out) {
  extern __shared__ float cb_sm[];
  const int hw = H * W;
  float* avg = cb_sm;            // [C]
  float* mx = avg + C;           // [C]
  float* cg = mx + C;            // [C]
  float* hid = cg + C;           // [2 R]
  float* comp = hid + 2 * R;     // [2 hw]: max over channels, mean over channels
  float* sg = comp + 2 * hw;     // [hw]
  const long long base = (long long)blockIdx.x * hw * C;
  const float* yf = y + base;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f, m = -INFINITY;
    for (int p = 0; p < hw; ++p) {
      const float v = yf[(long long)p * C + c];
      s += v;
      m = fmaxf(m, v);
    }
    avg[c] = s / (float)hw;
    mx[c] = m;
  }
  __syncthreads();
  for (int j = warp; j < 2 * R; j += nwarp) {   // rows 0..R-1: the avg input; R..2R-1: the max input
    const float* in = j < R ? avg : mx;
    const float* wr = w1 + (long long)(j % R) * C;
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a = fmaf(__ldg(wr + c), in[c], a);
    a = warp_sum(a);
    if (lane == 0) hid[j] = fmaxf(a + __ldg(b1 + j % R), 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 2.f * __ldg(b2 + c);   // the second Linear's bias enters once per pooled input
    for (int j = 0; j < R; ++j) a = fmaf(__ldg(w2 + (long long)c * R + j), hid[j] + hid[R + j], a);
    cg[c] = 1.0f / (1.0f + expf(-a));
  }
  __syncthreads();
  for (int p = warp; p < hw; p += nwarp) {
    float m = -INFINITY, s = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float v = yf[(long long)p * C + c] * cg[c];
      m = fmaxf(m, v);
      s += v;
    }
    m = warp_max(m);
    s = warp_sum(s);
    if (lane == 0) {
      comp[p] = m;
      comp[hw + p] = s / (float)C;
    }
  }
  __syncthreads();
  for (int p = threadIdx.x; p < hw; p += blockDim.x) {
    const int py = p / W, px = p % W;
    float a = __ldg(bsp);
    for (int ch = 0; ch < 2; ++ch)
      for (int ky = 0; ky < 7; ++ky) {
        const int iy = py + ky - 3;
        if (iy < 0 || iy >= H) continue;
        for (int kx = 0; kx < 7; ++kx) {
          const int ix = px + kx - 3;
          if (ix >= 0 && ix < W) a = fmaf(__ldg(wsp + (ch * 7 + ky) * 7 + kx), comp[ch * hw + iy * W + ix], a);
        }
      }
    sg[p] = 1.0f / (1.0f + expf(-a));
  }
  __syncthreads();
  const float* rf = res + base;
  float* of = out + base;
  for (long long i = threadIdx.x; i < (long long)hw * C; i += blockDim.x) {
    const int c = (int)(i % C), p = (int)(i / C);
    of[i] = fmaxf(fmaf(yf[i] * cg[c], sg[p], rf[i]), 0.f);
  }
}

// out[n, c0 + c] (+)= mean_hw(x[n, :, c]) / div   (one block per frame)
__global__ void __launch_bounds__(256)
gap_kernel(const float* __restrict__ x, int hw, int C, int Cs, float* __restrict__ out, int ld_out, int c0, int accumulate,
           float inv) {
  const long long n = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < hw; ++p) s += x[(n * hw + p) * Cs + c];
    float* o = out + n * ld_out + c0 + c;
    const float v = s * inv;
    *o = accumulate ? *o + v : v;
  }
}

// dst[r, j] = act(src[r, s0 + j] * a[j] + b[j]) for j < C (pre-activation BatchNorm of EmoNet's ConvBlocks); 4 channels
// per thread, dst rows are C wide
__global__ void __launch_bounds__(256)
affine_kernel(const float* __restrict__ src, int s_ld, int s0, const float4* __restrict__ a, const float4* __restrict__ b,
              float4* __restrict__ dst, int c4, int relu, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int j = (int)(idx % c4);
  const long long r = idx / c4;
  const float4 v = __ldg(reinterpret_cast<const float4*>(src + r * s_ld + s0) + j), sa = __ldg(a + j), sb = __ldg(b + j);
  float4 o = make_float4(fmaf(v.x, sa.x, sb.x), fmaf(v.y, sa.y, sb.y), fmaf(v.z, sa.z, sb.z), fmaf(v.w, sa.w, sb.w));
  if (relu) o = make_float4(fmaxf(o.x, 0.f), fmaxf(o.y, 0.f), fmaxf(o.z, 0.f), fmaxf(o.w, 0.f));
  dst[idx] = o;
}

// dst = big + nearest-neighbour x2 upsample of small (F.interpolate(scale_factor=2)); big / dst are [n, 2h, 2w, c]
__global__ void __launch_bounds__(256)
upadd_kernel(const float4* __restrict__ big, const float4* __restrict__ small, int h2, int w2, int c4,
             float4* __restrict__ dst, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = (int)(idx % c4);
  const long long pos = idx / c4;
  const int x = (int)(pos % w2), y = (int)((pos / w2) % h2);
  const long long n = pos / ((long long)w2 * h2);
  const float4 a = __ldg(big + idx), s = __ldg(small + ((n * (h2 / 2) + y / 2) * (w2 / 2) + x / 2) * (long long)c4 + c);
  dst[idx] = make_float4(a.x + s.x, a.y + s.y, a.z + s.z, a.w + s.w);
}

// dst[r, d0 + j] = src[r, s0 + j] * sum_{c < mc} mask[r, c]   (EmoNet: features times the summed heat-maps);
// one warp per row
__global__ void __launch_bounds__(256)
maskmul_kernel(const float* __restrict__ src, int s_ld, int s0, const float* __restrict__ mask, int m_ld, int mc,
               float* __restrict__ dst, int d_ld, int d0, int width, long long rows) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  float m = 0.f;
  for (int c = lane; c < mc; c += 32) m += mask[r * m_ld + c];
  m = warp_sum(m);
  for (int j = lane; j < width; j += 32) dst[r * d_ld + d0 + j] = src[r * s_ld + s0 + j] * m;
}

struct CnnPlan { long long off_buf[CNN_BUFS], off_col, off_cu, off_z, off_scale, total; };

// torch MaxPool2d(3, 2, pad, ceil_mode) output size (pooling_output_shape: floor division); < 1 where torch raises
// (pad 0 with in = 1, or in = 2 in floor mode: the window does not fit)
int pool_out(int in, int pad, int ceil_mode) {
  const int num = in + 2 * pad - 3 + (ceil_mode ? 1 : 0);
  int o = (num >= 0 ? num / 2 : -((1 - num) / 2)) + 1;
  if (ceil_mode && (o - 1) * 2 >= in + pad) --o;  // the last window must start inside the (left-padded) input
  return o;
}

// One pass over the op table.  exec == false: shape inference + buffer extents (cnn_plan); exec == true: launches.
int cnn_walk(const MerCnnModel* m, int n_frames, bool exec, CnnPlan* plan, char* ws, const uint8_t* frames_bgr,
             float* out_feats, cudaStream_t st) {
  MER_REQUIRE(m && m->convs && m->ops && m->n_ops > 0 && m->n_convs > 0, "mer_cnn: empty model");
  MER_REQUIRE(m->gemm_mode == MER_GEMM_F16 || m->gemm_mode == MER_GEMM_BF16X3, "mer_cnn: gemm_mode %d", m->gemm_mode);
  const long long n = n_frames;
  const bool split = m->gemm_mode == MER_GEMM_BF16X3;
  const long long vbytes = split ? 4 : 2;  // bytes per operand value
  Shape sh[CNN_BUFS] = {};
  long long need[CNN_BUFS] = {}, col_need = 0;
  int se_c = 0, gaps = 0;
  float* buf[CNN_BUFS] = {};
  uint16_t* col = nullptr;
  int* offsets = nullptr;
  if (exec) {
    for (int b = 0; b < CNN_BUFS; ++b) buf[b] = reinterpret_cast<float*>(ws + plan->off_buf[b]);
    col = reinterpret_cast<uint16_t*>(ws + plan->off_col);
    offsets = reinterpret_cast<int*>(ws + plan->off_cu);
  }
  auto ok_buf = [](int b) { return b >= 0 && b < CNN_BUFS; };
  auto define = [&](int b, Shape s) {
    sh[b] = s;
    const long long fl = n * s.H * s.W * s.Cs;
    if (fl > need[b]) need[b] = fl;
  };
  for (int i = 0; i < m->n_ops; ++i) {
    const MerCnnOp& op = m->ops[i];
    MER_REQUIRE(ok_buf(op.dst) && ok_buf(op.src) && (op.res < 0 || ok_buf(op.res)), "mer_cnn: op %d buffer index", i);
    switch (op.kind) {
      case MER_CNN_STEM: {
        MER_REQUIRE(op.conv >= 0 && op.conv < m->n_convs, "mer_cnn: op %d conv index %d", i, op.conv);
        const MerResnetConv& cv = m->convs[op.conv];
        MER_REQUIRE(cv.k == 7 && cv.stride == 2 && cv.pad == 3 && cv.cin == 3 && cv.kpad == (split ? 160 : 192),
                    "mer_cnn: the stem is a 7x7 / 2 convolution packed to %d columns", split ? 160 : 192);
        MER_REQUIRE(cv.cout > 0 && cv.cout <= cv.cout_pad && cv.cout_pad % 128 == 0 && m->in_h > 0 && m->in_w > 0,
                    "mer_cnn: op %d stem geometry (cout %d stored as %d, frames %d x %d)", i, cv.cout, cv.cout_pad,
                    m->in_h, m->in_w);
        const int OH = (m->in_h + 6 - 7) / 2 + 1, OW = (m->in_w + 6 - 7) / 2 + 1;
        const long long rows = n * OH * OW, total = rows * cv.kpad;
        MER_REQUIRE(rows < (1ll << 31), "mer_cnn: too many frames per call");
        if (rows * cv.kpad * vbytes > col_need) col_need = rows * cv.kpad * vbytes;
        define(op.dst, Shape{OH, OW, cv.cout, cv.cout_pad});
        if (!exec) break;
        const unsigned blocks = (unsigned)((total + 255) / 256);
        if (split)
          im2col_stem_kernel<true><<<blocks, 256, 0, st>>>(frames_bgr, m->in_h, m->in_w, OH, OW, cv.kpad, m->scale,
                                                           m->mean[0], m->mean[1], m->mean[2], m->std[0], m->std[1],
                                                           m->std[2], col, total);
        else
          im2col_stem_kernel<false><<<blocks, 256, 0, st>>>(frames_bgr, m->in_h, m->in_w, OH, OW, cv.kpad, m->scale,
                                                            m->mean[0], m->mean[1], m->mean[2], m->std[0], m->std[1],
                                                            m->std[2], col, total);
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(1);
        MerGemmDesc g;
        memset(&g, 0, sizeof(g));
        g.A = reinterpret_cast<const float*>(col);
        g.W = static_cast<const float*>(cv.w);
        g.rows_per_batch = (int)rows;
        g.a_rows_dim = (int)rows;
        g.batches = 1;
        g.N = cv.cout_pad;
        g.K_inner = cv.kpad;
        g.taps = 1;
        g.P = 1;
        g.a_phase_stride = cv.kpad;
        g.a_row_stride = cv.kpad;
        g.a_batch_stride = rows * cv.kpad;
        g.mode = m->gemm_mode;
        g.ep.bias = cv.b;
        g.ep.out = buf[op.dst];
        g.ep.ld_out = cv.cout_pad;
        g.ep.flags = op.relu ? MER_EPI_RELU : 0;
        if (int rc = mer_gemm_launch(&g, st)) return rc;
        break;
      }
      case MER_CNN_CONV: {
        MER_REQUIRE(op.conv >= 0 && op.conv < m->n_convs, "mer_cnn: op %d conv index %d", i, op.conv);
        const MerResnetConv& cv = m->convs[op.conv];
        const Shape full = sh[op.src];
        const int c0 = op.p[0];  // the conv reads channels [c0, c0 + cin) of src
        MER_REQUIRE(full.H > 0 && c0 >= 0 && c0 % 4 == 0 && c0 + cv.cin <= full.C && op.src != op.dst,
                    "mer_cnn: op %d reads channels [%d, %d) of a %d-channel buffer", i, c0, c0 + cv.cin, full.C);
        // what conv() and mer_gemm_launch require, checked here so that a table they would refuse is refused by
        // mer_cnn_workspace_bytes and by mer_cnn_forward before its first launch
        const int K = cv.k * cv.k * cv.cin;
        MER_REQUIRE(cv.k > 0 && cv.stride > 0 && cv.pad >= 0 && cv.cin > 0 && cv.cin % 8 == 0 && cv.kpad == K &&
                        K % (split ? 32 : 64) == 0 && cv.cout > 0 && cv.cout <= cv.cout_pad && cv.cout_pad % 128 == 0,
                    "mer_cnn: op %d conv geometry (k %d stride %d pad %d, cin %d, kpad %d for K %d, cout %d stored as "
                    "%d)", i, cv.k, cv.stride, cv.pad, cv.cin, cv.kpad, K, cv.cout, cv.cout_pad);
        MER_REQUIRE(full.H + 2 * cv.pad >= cv.k && full.W + 2 * cv.pad >= cv.k,
                    "mer_cnn: op %d %dx%d conv (pad %d) of a %d x %d map", i, cv.k, cv.k, cv.pad, full.H, full.W);
        const Shape in{full.H, full.W, cv.cin, full.Cs};
        const int OH = (in.H + 2 * cv.pad - cv.k) / cv.stride + 1, OW = (in.W + 2 * cv.pad - cv.k) / cv.stride + 1;
        const long long rows = n * OH * OW;
        MER_REQUIRE(rows < (1ll << 31), "mer_cnn: too many frames per call");
        if (rows * cv.kpad * vbytes > col_need) col_need = rows * cv.kpad * vbytes;
        if (op.res >= 0)
          MER_REQUIRE(sh[op.res].H == OH && sh[op.res].W == OW && sh[op.res].Cs == cv.cout_pad,
                      "mer_cnn: op %d residual shape", i);
        if (exec) {
          Shape out;
          if (int rc = conv(cv, buf[op.src] + c0, in, n_frames, col, op.res >= 0 ? buf[op.res] : nullptr, op.relu != 0,
                            buf[op.dst], &out, st, m->gemm_mode))
            return rc;
        }
        define(op.dst, Shape{OH, OW, cv.cout, cv.cout_pad});
        break;
      }
      case MER_CNN_MAXPOOL: {
        const Shape in = sh[op.src];
        MER_REQUIRE(in.H > 0 && (op.k == 3 || op.k == 2) && op.stride == 2 && op.src != op.dst,
                    "mer_cnn: op %d max-pool", i);
        if (op.k == 2) {  // max_pool2d(x, 2, 2) on even maps
          MER_REQUIRE(in.H % 2 == 0 && in.W % 2 == 0 && op.pad == 0, "mer_cnn: op %d 2x2 max-pool of a %d x %d map", i,
                      in.H, in.W);
          define(op.dst, Shape{in.H / 2, in.W / 2, in.C, in.Cs});
          if (!exec) break;
          const long long total2 = n * (in.H / 2) * (in.W / 2) * (in.Cs / 4);
          maxpool2x2_kernel<<<(unsigned)((total2 + 255) / 256), 256, 0, st>>>(
              reinterpret_cast<const float4*>(buf[op.src]), in.H, in.W, in.Cs / 4, reinterpret_cast<float4*>(buf[op.dst]),
              total2);
          MER_CUDA_CHECK(cudaGetLastError());
          mer_count_launches(1);
          break;
        }
        const int OH = pool_out(in.H, op.pad, op.ceil_mode), OW = pool_out(in.W, op.pad, op.ceil_mode);
        MER_REQUIRE((op.pad == 0 || op.pad == 1) && OH > 0 && OW > 0,
                    "mer_cnn: op %d 3x3 max-pool (pad %d) of a %d x %d map", i, op.pad, in.H, in.W);
        define(op.dst, Shape{OH, OW, in.C, in.Cs});
        if (!exec) break;
        const long long total = n * OH * OW * (in.Cs / 4);
        maxpool3x3s2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
            reinterpret_cast<const float4*>(buf[op.src]), in.H, in.W, in.Cs / 4, OH, OW, op.pad,
            reinterpret_cast<float4*>(buf[op.dst]), total);
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(1);
        break;
      }
      case MER_CNN_SE: {
        const Shape in = sh[op.src];
        MER_REQUIRE(op.conv >= 0 && op.conv < m->n_convs && op.k >= 0 && op.k < m->n_convs, "mer_cnn: op %d SE layers", i);
        const MerResnetConv &dn = m->convs[op.conv], &up = m->convs[op.k];
        MER_REQUIRE(in.H > 0 && in.C == in.Cs && in.C % 4 == 0 && dn.cin == in.C && up.cout == in.C &&
                        dn.cout == up.cin && dn.cout > 0 && dn.cout <= 1024,
                    "mer_cnn: op %d SE geometry (C %d, %d -> %d -> %d)", i, in.C, dn.cin, dn.cout, up.cout);
        MER_REQUIRE(op.res >= 0 && sh[op.res].H == in.H && sh[op.res].W == in.W && sh[op.res].Cs == in.Cs,
                    "mer_cnn: op %d SE shortcut shape", i);
        if (in.C > se_c) se_c = in.C;
        define(op.dst, in);
        if (!exec) break;
        float* z = reinterpret_cast<float*>(ws + plan->off_z);
        float* scale = reinterpret_cast<float*>(ws + plan->off_scale);
        if (int rc = mer_iota_offsets_launch(offsets, n_frames, in.H * in.W, st)) return rc;
        if (int rc = mer_segment_reduce_launch(buf[op.src], offsets, offsets + 1, n_frames, in.C, MER_SEG_MEAN, z, st))
          return rc;
        se_mlp_kernel<<<n_frames, 256, (size_t)(in.C + dn.cout) * sizeof(float), st>>>(
            z, static_cast<const float*>(dn.w), dn.b, static_cast<const float*>(up.w), up.b, in.C, dn.cout, scale);
        MER_CUDA_CHECK(cudaGetLastError());
        const long long hw_c4 = (long long)in.H * in.W * (in.C / 4), total = hw_c4 * n_frames;
        se_apply_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
            reinterpret_cast<const float4*>(buf[op.src]), reinterpret_cast<const float4*>(buf[op.res]),
            reinterpret_cast<const float4*>(scale), hw_c4, in.C / 4, reinterpret_cast<float4*>(buf[op.dst]), total);
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(2);
        break;
      }
      case MER_CNN_CROP: {
        const Shape in = sh[op.src];
        const int y0 = op.p[0], x0 = op.p[1], h = op.p[2], w = op.p[3];
        MER_REQUIRE(in.H > 0 && op.src != op.dst && y0 >= 0 && x0 >= 0 && h > 0 && w > 0 && y0 + h <= in.H && x0 + w <= in.W,
                    "mer_cnn: op %d crop [%d:%d, %d:%d] of a %d x %d map", i, y0, y0 + h, x0, x0 + w, in.H, in.W);
        define(op.dst, Shape{h, w, in.C, in.Cs});
        if (!exec) break;
        const long long total = n * h * w * (in.Cs / 4);
        crop_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float4*>(buf[op.src]), in.H,
                                                                     in.W, in.Cs / 4, y0, x0, h, w,
                                                                     reinterpret_cast<float4*>(buf[op.dst]), total);
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(1);
        break;
      }
      case MER_CNN_SHAPE: {  // dst becomes an [H, W] map like src with p[0] channels (contents undefined)
        const Shape in = sh[op.src];
        MER_REQUIRE(in.H > 0 && op.p[0] > 0 && op.p[0] % 4 == 0, "mer_cnn: op %d shape", i);
        define(op.dst, Shape{in.H, in.W, op.p[0], op.p[0]});
        break;
      }
      case MER_CNN_SLICE: {
        const Shape a = sh[op.src], d = sh[op.dst];
        const int s0 = op.p[0], d0 = op.p[1], w = op.p[2], r0 = op.p[3];
        MER_REQUIRE(a.H > 0 && d.H == a.H && d.W == a.W && w > 0 && w % 4 == 0 && s0 % 4 == 0 && d0 % 4 == 0 &&
                        s0 >= 0 && d0 >= 0 && s0 + w <= a.Cs && d0 + w <= d.Cs,
                    "mer_cnn: op %d slice [%d, %d) -> [%d, %d)", i, s0, s0 + w, d0, d0 + w);
        if (op.res >= 0)
          MER_REQUIRE(sh[op.res].H == a.H && sh[op.res].W == a.W && r0 >= 0 && r0 % 4 == 0 && r0 + w <= sh[op.res].Cs,
                      "mer_cnn: op %d slice addend", i);
        if (!exec) break;
        const long long total = n * a.H * a.W * (w / 4);
        slice_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
            buf[op.src], a.Cs, s0, op.res >= 0 ? buf[op.res] : nullptr, op.res >= 0 ? sh[op.res].Cs : 0, r0, buf[op.dst],
            d.Cs, d0, w / 4, op.relu == 1, op.relu == 2, total);
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(1);
        break;
      }
      case MER_CNN_CBAM: {
        const Shape in = sh[op.src];
        MER_REQUIRE(op.conv >= 0 && op.conv < m->n_convs && op.p[0] >= 0 && op.p[0] < m->n_convs && op.p[1] >= 0 &&
                        op.p[1] < m->n_convs, "mer_cnn: op %d CBAM layers", i);
        const MerResnetConv &l1 = m->convs[op.conv], &l2 = m->convs[op.p[0]], &sp = m->convs[op.p[1]];
        MER_REQUIRE(in.H > 0 && in.C == in.Cs && in.H * in.W <= 64 && l1.cin == in.C && l2.cout == in.C &&
                        l1.cout == l2.cin && l1.cout <= 64 && sp.k == 7 && sp.cin == 2 && sp.cout == 1,
                    "mer_cnn: op %d CBAM geometry (%d x %d x %d)", i, in.H, in.W, in.C);
        MER_REQUIRE(op.res >= 0 && sh[op.res].H == in.H && sh[op.res].W == in.W && sh[op.res].Cs == in.Cs,
                    "mer_cnn: op %d CBAM shortcut shape", i);
        define(op.dst, in);
        if (!exec) break;
        const size_t smem = (size_t)(3 * in.C + 2 * l1.cout + 3 * in.H * in.W) * sizeof(float);
        cbam_kernel<<<n_frames, 256, smem, st>>>(buf[op.src], buf[op.res], static_cast<const float*>(l1.w), l1.b,
                                                 static_cast<const float*>(l2.w), l2.b, static_cast<const float*>(sp.w),
                                                 sp.b, in.H, in.W, in.C, l1.cout, buf[op.dst]);
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(1);
        break;
      }
      case MER_CNN_AFFINE: {
        const Shape in = sh[op.src];
        MER_REQUIRE(op.conv >= 0 && op.conv < m->n_convs, "mer_cnn: op %d affine layer", i);
        const MerResnetConv& af = m->convs[op.conv];
        const int s0 = op.p[0], Cc = af.cout;
        MER_REQUIRE(in.H > 0 && op.src != op.dst && Cc > 0 && Cc % 4 == 0 && s0 >= 0 && s0 % 4 == 0 && s0 + Cc <= in.Cs,
                    "mer_cnn: op %d affine over channels [%d, %d) of %d", i, s0, s0 + Cc, in.Cs);
        define(op.dst, Shape{in.H, in.W, Cc, Cc});
        if (!exec) break;
        const long long total = n * in.H * in.W * (Cc / 4);
        affine_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
            buf[op.src], in.Cs, s0, static_cast<const float4*>(af.w), reinterpret_cast<const float4*>(af.b),
            reinterpret_cast<float4*>(buf[op.dst]), Cc / 4, op.relu != 0, total);
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(1);
        break;
      }
      case MER_CNN_UPADD: {
        const Shape lo = sh[op.src];
        MER_REQUIRE(op.res >= 0 && lo.H > 0 && sh[op.res].H == 2 * lo.H && sh[op.res].W == 2 * lo.W &&
                        sh[op.res].Cs == lo.Cs && op.src != op.dst,
                    "mer_cnn: op %d upsample-add shapes", i);
        define(op.dst, sh[op.res]);
        if (!exec) break;
        const long long total = n * 4 * lo.H * lo.W * (lo.Cs / 4);
        upadd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
            reinterpret_cast<const float4*>(buf[op.res]), reinterpret_cast<const float4*>(buf[op.src]), 2 * lo.H, 2 * lo.W,
            lo.Cs / 4, reinterpret_cast<float4*>(buf[op.dst]), total);
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(1);
        break;
      }
      case MER_CNN_MASKMUL: {
        const Shape a = sh[op.src], d = sh[op.dst];
        const int s0 = op.p[0], d0 = op.p[1], w = op.p[2], mc = op.p[3];
        MER_REQUIRE(op.res >= 0 && a.H > 0 && d.H == a.H && d.W == a.W && sh[op.res].H == a.H && sh[op.res].W == a.W &&
                        w > 0 && s0 >= 0 && d0 >= 0 && s0 + w <= a.Cs && d0 + w <= d.Cs && mc > 0 && mc <= sh[op.res].Cs,
                    "mer_cnn: op %d mask-multiply", i);
        if (!exec) break;
        const long long rows = n * a.H * a.W;
        maskmul_kernel<<<(unsigned)((rows * 32 + 255) / 256), 256, 0, st>>>(buf[op.src], a.Cs, s0, buf[op.res],
                                                                            sh[op.res].Cs, mc, buf[op.dst], d.Cs, d0, w,
                                                                            rows);
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(1);
        break;
      }
      case MER_CNN_GAP: {
        const Shape in = sh[op.src];
        const int c0 = op.p[0], div = op.p[2] > 0 ? op.p[2] : 1;
        MER_REQUIRE(in.H > 0 && c0 >= 0 && c0 + in.C <= m->feat_dim, "mer_cnn: op %d pools %d channels into [%d, %d)", i,
                    in.C, c0, m->feat_dim);
        ++gaps;
        if (!exec) break;
        gap_kernel<<<n_frames, 256, 0, st>>>(buf[op.src], in.H * in.W, in.C, in.Cs, out_feats, m->feat_dim, c0,
                                             op.p[1] != 0, 1.0f / (float)(in.H * in.W * div));
        MER_CUDA_CHECK(cudaGetLastError());
        mer_count_launches(1);
        break;
      }
      default:
        MER_REQUIRE(false, "mer_cnn: op %d kind %d", i, op.kind);
    }
  }
  MER_REQUIRE(gaps > 0, "mer_cnn: the op table has no average pool (nothing is written to out_feats)");
  if (!exec) {
    auto al = [](long long x) { return (x + 255) & ~255ll; };
    long long o = 0;
    for (int b = 0; b < CNN_BUFS; ++b) {
      plan->off_buf[b] = o;
      o += al(need[b] * 4);
    }
    plan->off_col = o;   o += al(col_need);
    plan->off_cu = o;    o += al((n + 1) * 4);
    plan->off_z = o;     o += al(n * se_c * 4);
    plan->off_scale = o; o += al(n * se_c * 4);
    plan->total = o;
  }
  return 0;
}
}  // namespace

extern "C" {

long long mer_cnn_workspace_bytes(const MerCnnModel* m, int n_frames) {
  CnnPlan p;
  if (n_frames <= 0 || cnn_walk(m, n_frames, false, &p, nullptr, nullptr, nullptr, nullptr)) return -1;
  return p.total;
}

int mer_cnn_forward(const MerCnnModel* m, const uint8_t* frames_bgr, int n_frames, void* workspace,
                    long long workspace_bytes, float* out_feats, void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(m && frames_bgr && workspace && out_feats && n_frames > 0, "mer_cnn_forward: bad operands");
  CnnPlan p;
  if (int rc = cnn_walk(m, n_frames, false, &p, nullptr, nullptr, nullptr, nullptr)) return rc;
  MER_REQUIRE(workspace_bytes >= p.total, "mer_cnn_forward: workspace %lld B < required %lld B", workspace_bytes, p.total);
  return cnn_walk(m, n_frames, true, &p, static_cast<char*>(workspace), frames_bgr, out_feats, st);
}

}  // extern "C"
