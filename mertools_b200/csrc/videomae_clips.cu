// videomae_clips.cu — the MER2024 / MER2026 VideoMAE face-clip extractor (extract_sun_videomae.py:216-359).
//
// videomae_clips_kernel : S x S RGB uint8 frames + a table of 16 resolved frame rows per view -> the tubelet patch
//                         operand [n_views * tokens_per_view, 1536] of the Conv3d (2, 16, 16) / (2, 16, 16) patch
//                         embedding, columns in the weight's flatten order (c, dt, dy, dx), ClipToTensor + Normalize
//                         (volume_transforms.py, functional.py:76-88) computed in IEEE fp32 as the reference does
// mer_videomae_forward  : that operand -> patch GEMM (+ bias + sinusoid table) -> pre-LN stack -> final LayerNorm ->
//                         mean over each view's tokens (modeling_finetune.py VisionTransformer.forward_features with
//                         use_mean_pooling=False)
#include <cuda_fp16.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

constexpr int KPATCH = 1536;  // 3 channels x 2 frames x 16 x 16
constexpr int VEC = 8;        // columns per thread: one 16-byte fp16 store, two fp32 ones
constexpr int THREADS = KPATCH / VEC;

// One CTA per output row (token); thread j writes columns [8 j, 8 j + 8): channel c, frame dt of the tubelet, patch
// row dy, patch columns 8 (j & 1) .. + 8.  Consecutive threads write consecutive 16-byte chunks of the row.
// A row index outside [0, n_frames) is not read: the entries it would feed are NaN.
template <bool F32>
__global__ void __launch_bounds__(THREADS)
videomae_clips_kernel(const uint8_t* __restrict__ frames, int n_frames, int S, const int* __restrict__ rows,
                      void* __restrict__ out, float m0, float m1, float m2, float s0, float s1, float s2) {
  const int g = S / 16;
  const int per_t = g * g;
  const long long row = blockIdx.x;
  const int tok = (int)(row % (8 * per_t));
  const long long view = row / (8 * per_t);
  const int t = tok / per_t, py = (tok % per_t) / g, px = tok % g;
  const int j = threadIdx.x;
  const int c = j >> 6, dt = (j >> 5) & 1, dy = (j >> 1) & 15, dx0 = (j & 1) * 8;
  const int fr = __ldg(rows + view * 16 + 2 * t + dt);
  const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
  float v[VEC];
  if (fr >= 0 && fr < n_frames) {
    const uint8_t* src = frames + (((long long)fr * S + py * 16 + dy) * S + px * 16 + dx0) * 3 + c;
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = ((float)__ldg(src + 3 * i) / 255.0f - mean) / sd;
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = __int_as_float(0x7fc00000);
  }
  if (F32) {
    float4* o = reinterpret_cast<float4*>(static_cast<float*>(out) + row * KPATCH + j * VEC);
    o[0] = make_float4(v[0], v[1], v[2], v[3]);
    o[1] = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    uint4 pk;
    __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
    __half2 h2 = __floats2half2_rn(v[4], v[5]), h3 = __floats2half2_rn(v[6], v[7]);
    pk.x = *reinterpret_cast<uint32_t*>(&h0);
    pk.y = *reinterpret_cast<uint32_t*>(&h1);
    pk.z = *reinterpret_cast<uint32_t*>(&h2);
    pk.w = *reinterpret_cast<uint32_t*>(&h3);
    *reinterpret_cast<uint4*>(static_cast<__half*>(out) + row * KPATCH + j * VEC) = pk;
  }
}

// ImageNet mean / std of video_transforms.Normalize as the fp32 values torch.as_tensor gives them
constexpr float kMean[3] = {0.485f, 0.456f, 0.406f};
constexpr float kStd[3] = {0.229f, 0.224f, 0.225f};

int clips_launch(const uint8_t* frames, int n_frames, int S, const int* rows, int n_views, void* out, bool f32,
                 cudaStream_t stream) {
  const long long n_rows = (long long)n_views * 8 * (S / 16) * (S / 16);
  MER_REQUIRE(n_rows < (1ll << 31), "mer_videomae_clips: %lld rows", n_rows);
  if (f32)
    videomae_clips_kernel<true><<<(unsigned)n_rows, THREADS, 0, stream>>>(frames, n_frames, S, rows, out, kMean[0],
                                                                          kMean[1], kMean[2], kStd[0], kStd[1], kStd[2]);
  else
    videomae_clips_kernel<false><<<(unsigned)n_rows, THREADS, 0, stream>>>(frames, n_frames, S, rows, out, kMean[0],
                                                                           kMean[1], kMean[2], kStd[0], kStd[1], kStd[2]);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

#define MER_TRY(expr)                 \
  do {                                \
    if (int _rc = (expr)) return _rc; \
  } while (0)

struct Plan { long long M, vt_ld, off_x, off_xn, off_qkv, off_h, off_vt, off_cu, off_rows, total; int tpv; };

Plan plan(const MerVideoMaeModel* m, int n_views) {
  Plan p;
  const int g = m->img / 16;
  p.tpv = 8 * g * g;
  p.M = (long long)n_views * p.tpv;
  p.vt_ld = (p.M + 7) & ~7ll;
  auto al = [](long long x) { return (x + 255) & ~255ll; };
  const long long D = m->dim;
  long long o = 0;
  p.off_x = o;    o += al(p.M * D * 4);
  p.off_xn = o;   o += al(p.M * D * 4);
  p.off_qkv = o;  o += al(p.M * 3 * D * 4);
  const long long hb = p.M * (long long)m->ffn * 4, pb = p.M * KPATCH * 2;
  p.off_h = o;    o += al(hb > pb ? hb : pb);  // FFN buffer; the fp16 patch operand lives here first
  p.off_vt = o;   o += al(D * p.vt_ld * 4);
  p.off_cu = o;   o += al(((long long)n_views + 1) * 4);
  p.off_rows = o; o += al((long long)n_views * 16 * 4);
  p.total = o;
  return p;
}

int check_model(const MerVideoMaeModel* m) {
  MER_REQUIRE(m && m->patch_w && m->patch_b && m->pos && m->layers && m->norm_g && m->norm_b,
              "mer_videomae: null model operand");
  MER_REQUIRE(m->n_layers >= 1 && m->heads >= 1 && m->heads * 64 == m->dim,
              "mer_videomae: heads %d x 64 != dim %d (or n_layers %d < 1)", m->heads, m->dim, m->n_layers);
  MER_REQUIRE(m->dim == 384 || m->dim == 512 || m->dim == 768 || m->dim == 1024 || m->dim == 1280 || m->dim == 1536,
              "mer_videomae: dim %d is not a LayerNorm width", m->dim);
  MER_REQUIRE(m->ffn >= 768 && m->ffn % 128 == 0, "mer_videomae: ffn %d", m->ffn);
  // 800 / 1568 tokens per view: the fp16 V^T attention's long rows (254 .. MER_ATT_LONG_MAX)
  MER_REQUIRE(m->img == 160 || m->img == 224, "mer_videomae: img %d (160 or 224)", m->img);
  return 0;
}

}  // namespace

extern "C" {

int mer_videomae_clips(const uint8_t* frames, int n_frames, int S, const int32_t* view_rows, int n_views, void* out,
                       int out_f32, void* stream) {
  MER_REQUIRE(frames && view_rows && out, "mer_videomae_clips: null operand");
  MER_REQUIRE(n_frames > 0 && n_views > 0, "mer_videomae_clips: n_frames %d, n_views %d", n_frames, n_views);
  MER_REQUIRE(S == 160 || S == 224, "mer_videomae_clips: S %d (160 or 224)", S);
  return clips_launch(frames, n_frames, S, view_rows, n_views, out, out_f32 != 0, static_cast<cudaStream_t>(stream));
}

long long mer_videomae_workspace_bytes(const MerVideoMaeModel* m, int n_views) {
  if (check_model(m) || n_views <= 0) return -1;
  return plan(m, n_views).total;
}

int mer_videomae_forward(const MerVideoMaeModel* m, const uint8_t* frames, int n_frames, const int32_t* view_rows,
                         int n_views, void* workspace, long long workspace_bytes, float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_TRY(check_model(m));
  MER_REQUIRE(frames && view_rows && workspace && out, "mer_videomae_forward: null operand");
  MER_REQUIRE(n_frames > 0 && n_views > 0, "mer_videomae_forward: n_frames %d, n_views %d", n_frames, n_views);
  const Plan p = plan(m, n_views);
  MER_REQUIRE(workspace_bytes >= p.total, "mer_videomae_forward: workspace %lld B < required %lld B", workspace_bytes,
              p.total);
  MER_REQUIRE(p.M * 3 * m->dim < (1ll << 31), "mer_videomae_forward: too many views (%d)", n_views);
  for (long long i = 0; i < (long long)n_views * 16; ++i)
    MER_REQUIRE(view_rows[i] >= 0 && view_rows[i] < n_frames, "mer_videomae_forward: view %lld row %d not in [0, %d)",
                i / 16, view_rows[i], n_frames);
  char* ws = static_cast<char*>(workspace);
  float* x = reinterpret_cast<float*>(ws + p.off_x);
  float* xn = reinterpret_cast<float*>(ws + p.off_xn);
  float* qkv = reinterpret_cast<float*>(ws + p.off_qkv);
  float* h = reinterpret_cast<float*>(ws + p.off_h);
  float* vt = reinterpret_cast<float*>(ws + p.off_vt);
  int* offsets = reinterpret_cast<int*>(ws + p.off_cu);
  int* rows = reinterpret_cast<int*>(ws + p.off_rows);
  const int D = m->dim;

  MER_CUDA_CHECK(cudaMemcpyAsync(rows, view_rows, (size_t)n_views * 16 * 4, cudaMemcpyHostToDevice, stream));
  MER_TRY(mer_iota_offsets_launch(offsets, n_views, p.tpv, stream));
  MER_TRY(clips_launch(frames, n_frames, m->img, rows, n_views, h, false, stream));
  {
    MerGemmDesc g;
    memset(&g, 0, sizeof(g));
    g.A = h;
    g.W = static_cast<const float*>(m->patch_w);
    g.rows_per_batch = p.tpv;
    g.a_rows_dim = p.tpv;
    g.batches = n_views;
    g.N = D;
    g.K_inner = KPATCH;
    g.taps = 1;
    g.P = 1;
    g.a_phase_stride = KPATCH;
    g.a_row_stride = KPATCH;
    g.a_batch_stride = (long long)p.tpv * KPATCH;
    g.ep.bias = m->patch_b;
    g.ep.res = m->pos;  // + the sinusoid table, same for every view
    g.ep.res_bstride = 0;
    g.ep.out = x;
    g.ep.out_bstride = p.tpv;
    g.ep.ld_out = D;
    g.ep.ld_res = D;
    g.mode = MER_GEMM_F16;
    MER_TRY(mer_gemm_launch(&g, stream));
  }
  MerStackArgs a;
  memset(&a, 0, sizeof(a));
  a.layers = m->layers;
  a.n_layers = m->n_layers;
  a.pre_ln = 1;
  a.mode = MER_GEMM_F16;
  a.dim = D;
  a.ffn = m->ffn;
  a.heads = m->heads;
  a.eps = m->ln_eps;
  a.tokens = p.M;
  a.cu_seqlens = offsets;
  a.n_seq = n_views;
  a.max_seqlen = p.tpv;
  a.x = x;
  a.xn = xn;
  a.qkv = qkv;
  a.h = h;
  a.vt = vt;
  a.vt_ld = p.vt_ld;
  a.long_rows = 1;  // 800 / 1568-token rows: the fp16 V^T kernel
  MER_TRY(mer_run_stack(a, stream));
  MER_TRY(mer_layernorm_launch(x, m->norm_g, m->norm_b, xn, nullptr, nullptr, p.M, D, m->ln_eps, 0, stream));
  return mer_segment_reduce_launch(xn, offsets, offsets + 1, n_views, D, MER_SEG_MEAN, out, stream);
}

}  // extern "C"
