// fusion.cu — the Attention-fusion network of MERBench/toolkit/models/attention.py:8-57 (with
// MLPEncoder, modules/encoder.py:9-41), its loss (toolkit/utils/loss.py:5-28), the backward pass
// and the Adam update (main-release.py:50-66,205: torch.optim.Adam(lr, weight_decay=l2), optional
// clip_grad_value_), as explicit fp32 kernels.
//
// This is the tiny-kernel regime (0.48 MMAC per clip forward): everything is fp32 SIMT with a
// FIXED summation order (no atomics -> bit-reproducible), batched across the three modality
// encoders per launch, and the host captures the whole step in one CUDA graph.  The flat parameter
// / gradient buffers use the reference's state_dict order so the gradient buffer is the single
// NCCL all-reduce operand (477,962 floats at hidden 128).
#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

struct LinP {          // y = relu?( (x .* mask * mscale) W^T + b )
  const float* x; int ldx;
  const float* mask;   // dropout keep-mask (0/1) on x, or null
  float mscale;
  const float* W;      // [N,K]
  const float* b;      // [N]
  float* y; int ldy;
  int K, N, relu;
};
struct LinBatch { LinP p[3]; };

constexpr int KC = 128;

// grid (ceil(N/8), ceil(B/32), nprob); block 256: warp w -> output column, lane -> batch row
__global__ void __launch_bounds__(256)
fus_linear_fwd_kernel(const LinBatch lb, int B) {
  __shared__ float xs[KC][33];
  const LinP& p = lb.p[blockIdx.z];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + warp;
  const int b0 = blockIdx.y * 32;
  if (blockIdx.x * 8 >= p.N) return;
  float acc = 0.f;
  for (int k0 = 0; k0 < p.K; k0 += KC) {
    const int kc = min(KC, p.K - k0);
    for (int i = threadIdx.x; i < 32 * KC; i += 256) {
      const int r = i / KC, k = i % KC;
      float v = 0.f;
      if (b0 + r < B && k < kc) {
        v = p.x[(long long)(b0 + r) * p.ldx + k0 + k];
        if (p.mask) v *= p.mask[(long long)(b0 + r) * p.K + k0 + k] * p.mscale;
      }
      xs[k][r] = v;
    }
    __syncthreads();
    if (n < p.N) {
      const float* w = p.W + (long long)n * p.K + k0;
      for (int k = 0; k < kc; ++k) acc = fmaf(xs[k][lane], __ldg(w + k), acc);
    }
    __syncthreads();
  }
  if (n < p.N && b0 + lane < B) {
    float v = acc + p.b[n];
    if (p.relu) v = fmaxf(v, 0.f);
    p.y[(long long)(b0 + lane) * p.ldy + n] = v;
  }
}

struct BwdP {
  const float* dy; int lddy;   // grad wrt y (post-relu)
  const float* yact; int ldy;  // y itself (relu mask source) or null
  const float* x; int ldx;     // layer input (pre-dropout)
  const float* mask; float mscale;
  const float* W;
  float* dW; float* db;        // [N,K], [N]
  float* dx; int lddx;         // grad wrt x (null to skip)
  int accumulate_dx;
  int K, N;
};
struct BwdBatch { BwdP p[3]; };

// dW[n,k] = sum_b dyeff[b,n] * xd[b,k];  db[n] = sum_b dyeff[b,n].   grid (ceil(K/256), N, nprob)
__global__ void __launch_bounds__(256)
fus_linear_bwd_w_kernel(const BwdBatch bb, int B) {
  const BwdP& p = bb.p[blockIdx.z];
  const int n = blockIdx.y;
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (n >= p.N || blockIdx.x * 256 >= p.K) return;
  float acc = 0.f, accb = 0.f;
  for (int b = 0; b < B; ++b) {
    float g = p.dy[(long long)b * p.lddy + n];
    if (p.yact && !(p.yact[(long long)b * p.ldy + n] > 0.f)) g = 0.f;
    accb += g;
    if (k < p.K) {
      float xv = p.x[(long long)b * p.ldx + k];
      if (p.mask) xv *= p.mask[(long long)b * p.K + k] * p.mscale;
      acc = fmaf(g, xv, acc);
    }
  }
  if (k < p.K) p.dW[(long long)n * p.K + k] = acc;
  if (k == 0) p.db[n] = accb;
}

// dx[b,k] (+)= (sum_n dyeff[b,n] W[n,k]) * mask.   grid (ceil(K/256), B, nprob)
__global__ void __launch_bounds__(256)
fus_linear_bwd_x_kernel(const BwdBatch bb, int B) {
  __shared__ float dys[256];
  const BwdP& p = bb.p[blockIdx.z];
  if (!p.dx || blockIdx.x * 256 >= p.K) return;
  const int b = blockIdx.y;
  const int k = blockIdx.x * 256 + threadIdx.x;
  for (int n = threadIdx.x; n < p.N; n += 256) {
    float g = p.dy[(long long)b * p.lddy + n];
    if (p.yact && !(p.yact[(long long)b * p.ldy + n] > 0.f)) g = 0.f;
    dys[n] = g;
  }
  __syncthreads();
  if (k >= p.K) return;
  float acc = 0.f;
  for (int n = 0; n < p.N; ++n) acc = fmaf(dys[n], __ldg(p.W + (long long)n * p.K + k), acc);
  if (p.mask) acc *= p.mask[(long long)b * p.K + k] * p.mscale;
  float* d = p.dx + (long long)b * p.lddx + k;
  *d = p.accumulate_dx ? (*d + acc) : acc;
}

__device__ __forceinline__ float block_sum128(float v, float* sh) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  return (sh[0] + sh[1]) + (sh[2] + sh[3]);
}

struct HeadArgs {
  const float* h3cat;  // [B,3H]  audio | text | video hidden
  const float* a3;     // [B,H]   attention_mlp output
  const float* w_att; const float* b_att;  // [3,H],[3]
  const float* w_o1; const float* b_o1;    // [O1,H]
  const float* w_o2; const float* b_o2;    // [O2,H]
  const long long* emo; const float* val;  // labels or null (eval)
  float* features; float* emos_out; float* vals_out;  // [B,H],[B,O1],[B,O2]
  float* loss_terms;   // [B,2]
  float* d_emos; float* d_vals; float* d_att; float* d_cat; float* d_a3;
  int H, O1, O2;
  float inv_batch;     // 1 / (batch the loss is averaged over)
};

// one block (128 threads) per sample; H <= 256
__global__ void __launch_bounds__(128)
fus_head_kernel(const HeadArgs a) {
  __shared__ float sh[4];
  __shared__ float fused[256], dfused[256];
  __shared__ float att[3], datt[3], logits[16], dlog[16], dval[4];
  const int b = blockIdx.x, H = a.H, tid = threadIdx.x;
  const float* h3 = a.h3cat + (long long)b * 3 * H;
  const float* a3 = a.a3 + (long long)b * H;
  for (int m = 0; m < 3; ++m) {
    float s = 0.f;
    for (int j = tid; j < H; j += 128) s = fmaf(a.w_att[m * H + j], a3[j], s);
    s = block_sum128(s, sh);
    if (tid == 0) att[m] = s + a.b_att[m];
  }
  __syncthreads();
  for (int j = tid; j < H; j += 128) {
    const float f = (h3[j] * att[0] + h3[H + j] * att[1]) + h3[2 * H + j] * att[2];
    fused[j] = f;
    a.features[(long long)b * H + j] = f;
  }
  __syncthreads();
  for (int c = 0; c < a.O1; ++c) {
    float s = 0.f;
    for (int j = tid; j < H; j += 128) s = fmaf(a.w_o1[c * H + j], fused[j], s);
    s = block_sum128(s, sh);
    if (tid == 0) { logits[c] = s + a.b_o1[c]; a.emos_out[(long long)b * a.O1 + c] = logits[c]; }
  }
  for (int c = 0; c < a.O2; ++c) {
    float s = 0.f;
    for (int j = tid; j < H; j += 128) s = fmaf(a.w_o2[c * H + j], fused[j], s);
    s = block_sum128(s, sh);
    if (tid == 0) { dval[c] = s + a.b_o2[c]; a.vals_out[(long long)b * a.O2 + c] = dval[c]; }
  }
  __syncthreads();
  if (!a.emo) return;  // eval: forward only
  if (tid == 0) {
    // CELoss: NLL(log_softmax) summed / N ; MSELoss: squared error summed / N  (loss.py:11-28)
    float mx = logits[0];
    for (int c = 1; c < a.O1; ++c) mx = fmaxf(mx, logits[c]);
    float se = 0.f;
    for (int c = 0; c < a.O1; ++c) se += expf(logits[c] - mx);
    const float lse = mx + logf(se);
    const int tgt = (int)a.emo[b];
    a.loss_terms[2 * b + 0] = lse - logits[tgt];
    for (int c = 0; c < a.O1; ++c) {
      const float sm = expf(logits[c] - lse);
      dlog[c] = (sm - (c == tgt ? 1.f : 0.f)) * a.inv_batch;
      a.d_emos[(long long)b * a.O1 + c] = dlog[c];
    }
    float mse = 0.f;
    for (int c = 0; c < a.O2; ++c) {
      const float d = dval[c] - a.val[(long long)b * a.O2 + c];
      mse += d * d;
      dval[c] = 2.f * d * a.inv_batch;
      a.d_vals[(long long)b * a.O2 + c] = dval[c];
    }
    a.loss_terms[2 * b + 1] = mse;
  }
  __syncthreads();
  for (int j = tid; j < H; j += 128) {
    float s = 0.f;
    for (int c = 0; c < a.O1; ++c) s = fmaf(a.w_o1[c * H + j], dlog[c], s);
    for (int c = 0; c < a.O2; ++c) s = fmaf(a.w_o2[c * H + j], dval[c], s);
    dfused[j] = s;
  }
  __syncthreads();
  for (int m = 0; m < 3; ++m) {
    float s = 0.f;
    for (int j = tid; j < H; j += 128) s = fmaf(h3[m * H + j], dfused[j], s);
    s = block_sum128(s, sh);
    if (tid == 0) { datt[m] = s; a.d_att[3 * b + m] = s; }
  }
  __syncthreads();
  for (int j = tid; j < H; j += 128) {
    for (int m = 0; m < 3; ++m) a.d_cat[(long long)b * 3 * H + m * H + j] = att[m] * dfused[j];
    a.d_a3[(long long)b * H + j] =
        (a.w_att[j] * datt[0] + a.w_att[H + j] * datt[1]) + a.w_att[2 * H + j] * datt[2];
  }
}

__global__ void fus_loss_reduce_kernel(const float* terms, int B, float inv_batch, float* loss_out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float ce = 0.f, mse = 0.f;
  for (int b = 0; b < B; ++b) { ce += terms[2 * b]; mse += terms[2 * b + 1]; }
  loss_out[0] = ce * inv_batch;
  loss_out[1] = mse * inv_batch;
  loss_out[2] = ce * inv_batch + mse * inv_batch;
}

// torch.optim.Adam (coupled L2) in its own operation order; step counter lives on the device so a
// captured CUDA graph advances it on every replay.
__global__ void __launch_bounds__(256)
fus_adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                float* __restrict__ v, long long n, float lr, float beta1, float beta2, float eps,
                float wd, float gscale, float clip, const int* __restrict__ step) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float t = (float)(*step + 1);
  const float bc1 = 1.f - powf(beta1, t);
  const float bc2_sqrt = sqrtf(1.f - powf(beta2, t));
  float grad = g[i] * gscale;
  if (clip > 0.f) grad = fminf(fmaxf(grad, -clip), clip);
  float mi = m[i], vi = v[i];
  p[i] = mer::adam_param(p[i], grad, mi, vi, lr, beta1, beta2, eps, wd, bc1, bc2_sqrt);
  m[i] = mi;
  v[i] = vi;
}
__global__ void fus_step_inc_kernel(int* step) { if (threadIdx.x == 0 && blockIdx.x == 0) ++(*step); }

// keep-mask (0/1 floats) from a counter hash of (seed, step, index); keep prob = 1 - p
__global__ void __launch_bounds__(256)
fus_dropout_mask_kernel(float* mask, long long n, float p, unsigned long long seed, const int* step) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (unsigned long long)(*step + 1) +
                         0xD1B54A32D192ED03ull * (unsigned long long)(i + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  const float u = (float)(z >> 40) * (1.0f / 16777216.0f);
  mask[i] = u >= p ? 1.f : 0.f;
}

int check_dims(const MerFusionDims* d, int B) {
  MER_REQUIRE(d && d->hidden > 0 && d->hidden <= 256 && d->out1 > 0 && d->out1 <= 16 &&
                  d->out2 > 0 && d->out2 <= 4 && d->audio_dim > 0 && d->text_dim > 0 &&
                  d->video_dim > 0,
              "mer_fusion: unsupported dims (hidden <= 256, out1 <= 16, out2 <= 4)");
  MER_REQUIRE(B > 0 && B <= 65535, "mer_fusion: batch %d out of range", B);
  return 0;
}

// ================================================================================================
// Frame-level fusion (feat_type = frm_align / frm_unalign): LSTMEncoder (modules/encoder.py:45-72) per
// modality -- nn.LSTM(in, H, 1 layer, batch_first) over the zero-pre-padded sequence, final hidden state,
// dropout, Linear(H, H) -- feeding the same attention head.  fp32 throughout, fixed summation order.
// ================================================================================================
constexpr int LSTM_MAXH = 128;  // one W_hh row (H floats) lives in the registers of each gate thread

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// One block per batch row, 4H threads: thread j = gate row j of torch's (i, f, g, o) stacking.
// xw: [B, T, 4H] = x W_ih^T + b_ih (precomputed).  Writes the ACTIVATED gates, the cell state, the hidden
// state after and before each step (the backward pass and the weight gradients read them).
__global__ void __launch_bounds__(4 * LSTM_MAXH)
lstm_fwd_kernel(const float* __restrict__ xw, const float* __restrict__ w_hh, const float* __restrict__ b_hh,
                int T, int H, float* __restrict__ gates, float* __restrict__ cs, float* __restrict__ hs,
                float* __restrict__ hprev, float* __restrict__ h_last) {
  __shared__ float h_s[LSTM_MAXH];
  __shared__ float g_s[4 * LSTM_MAXH];
  const int b = blockIdx.x, j = threadIdx.x;
  float w[LSTM_MAXH];
#pragma unroll
  for (int k = 0; k < LSTM_MAXH; ++k) w[k] = k < H ? w_hh[(long long)j * H + k] : 0.f;
  const float bj = b_hh[j];
  const int type = j / H;
  float c = 0.f;
  if (j < H) h_s[j] = 0.f;
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    const long long row = (long long)b * T + t;
    float pre = xw[row * 4 * H + j] + bj;
#pragma unroll
    for (int k = 0; k < LSTM_MAXH; ++k)
      if (k < H) pre = fmaf(w[k], h_s[k], pre);
    const float act = type == 2 ? tanhf(pre) : sigmoidf_(pre);
    g_s[j] = act;
    gates[row * 4 * H + j] = act;
    __syncthreads();
    if (j < H) {
      hprev[row * H + j] = h_s[j];
      c = g_s[H + j] * c + g_s[j] * g_s[2 * H + j];
      const float h = g_s[3 * H + j] * tanhf(c);
      cs[row * H + j] = c;
      hs[row * H + j] = h;
      h_s[j] = h;
      if (t == T - 1) h_last[(long long)b * H + j] = h;
    }
    __syncthreads();
  }
}

// Back-propagation through time for one batch row: d_hT in, pre-activation gate gradients out.
// thread tid: unit k = tid % H; quarter q = tid / H holds W_hh[q*H + jj][k] (jj < H) for the
// dh_{t-1}[k] = sum_j W_hh[j][k] dpre[j] product, reduced over the four quarters through smem.
__global__ void __launch_bounds__(4 * LSTM_MAXH)
lstm_bwd_kernel(const float* __restrict__ d_hT, const float* __restrict__ w_hh, const float* __restrict__ gates,
                const float* __restrict__ cs, int T, int H, float* __restrict__ dgates) {
  __shared__ float dp_s[4 * LSTM_MAXH];
  __shared__ float part[4][LSTM_MAXH];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int k = tid % H, q = tid / H;
  float w[LSTM_MAXH];
#pragma unroll
  for (int jj = 0; jj < LSTM_MAXH; ++jj) w[jj] = jj < H ? w_hh[(long long)(q * H + jj) * H + k] : 0.f;
  float dh = tid < H ? d_hT[(long long)b * H + tid] : 0.f;
  float dc = 0.f;
  for (int t = T - 1; t >= 0; --t) {
    const long long row = (long long)b * T + t;
    if (tid < H) {
      const float* g = gates + row * 4 * H;
      const float gi = g[tid], gf = g[H + tid], gg = g[2 * H + tid], go = g[3 * H + tid];
      const float c = cs[row * H + tid];
      const float c_prev = t > 0 ? cs[(row - 1) * H + tid] : 0.f;
      const float tc = tanhf(c);
      const float d_o = dh * tc;
      dc += dh * go * (1.f - tc * tc);
      const float d_i = dc * gg, d_g = dc * gi, d_f = dc * c_prev;
      dc *= gf;
      const float pi = d_i * gi * (1.f - gi), pf = d_f * gf * (1.f - gf), pg = d_g * (1.f - gg * gg),
                  po = d_o * go * (1.f - go);
      dp_s[tid] = pi; dp_s[H + tid] = pf; dp_s[2 * H + tid] = pg; dp_s[3 * H + tid] = po;
      float* dg = dgates + row * 4 * H;
      dg[tid] = pi; dg[H + tid] = pf; dg[2 * H + tid] = pg; dg[3 * H + tid] = po;
    }
    __syncthreads();
    float acc = 0.f;
#pragma unroll
    for (int jj = 0; jj < LSTM_MAXH; ++jj)
      if (jj < H) acc = fmaf(w[jj], dp_s[q * H + jj], acc);
    part[q][k] = acc;
    __syncthreads();
    if (tid < H) dh = (part[0][tid] + part[1][tid]) + (part[2][tid] + part[3][tid]);
    __syncthreads();
  }
}

struct FrmLayout {  // reference state_dict order of Attention with LSTMEncoders (attention.py:25-33)
  long long w_ih[3], w_hh[3], b_ih[3], b_hh[3], lin_w[3], lin_b[3];
  long long att_w1, att_b1, att_w2, att_b2, att_w3, att_b3;
  long long fa_w, fa_b, o1_w, o1_b, o2_w, o2_b, total;
};

FrmLayout make_frm_layout(const MerFusionDims& d) {
  FrmLayout L;
  long long o = 0;
  const int in[3] = {d.audio_dim, d.text_dim, d.video_dim};
  const long long H = d.hidden;
  for (int m = 0; m < 3; ++m) {
    L.w_ih[m] = o; o += 4 * H * in[m];
    L.w_hh[m] = o; o += 4 * H * H;
    L.b_ih[m] = o; o += 4 * H;
    L.b_hh[m] = o; o += 4 * H;
    L.lin_w[m] = o; o += H * H;
    L.lin_b[m] = o; o += H;
  }
  L.att_w1 = o; o += H * 3 * H;
  L.att_b1 = o; o += H;
  L.att_w2 = o; o += H * H;
  L.att_b2 = o; o += H;
  L.att_w3 = o; o += H * H;
  L.att_b3 = o; o += H;
  L.fa_w = o; o += 3 * H;
  L.fa_b = o; o += 3;
  L.o1_w = o; o += (long long)d.out1 * H;
  L.o1_b = o; o += d.out1;
  L.o2_w = o; o += (long long)d.out2 * H;
  L.o2_b = o; o += d.out2;
  L.total = o;
  return L;
}

struct FrmScratch {
  float *xw[3], *gates[3], *dgates[3], *cs[3], *hs[3], *hprev[3];
  float *hT, *d_hT, *mask_h[3];      // [3][B,H]
  float *h3cat, *a1, *a2, *a3, *d_cat, *d_a1, *d_a2, *d_a3, *d_emos, *d_vals, *d_att, *loss_terms, *mask_cat;
};

long long frm_scratch_floats(const MerFusionDims& d, int B, const int T[3]) {
  const long long H = d.hidden;
  long long n = 0;
  for (int m = 0; m < 3; ++m) n += (long long)B * T[m] * (4 * H * 3 + H * 3);
  n += (long long)B * H * (3 + 3 + 3);                       // hT, d_hT, mask_h
  n += (long long)B * (3 * H + 3 * H + 3 * H + 3 * H + 3 * H)  // h3cat, a1..3, d_cat, d_a1..3, mask_cat
       + (long long)B * (d.out1 + d.out2 + 3 + 2);
  return n + 64;
}

FrmScratch frm_carve(const MerFusionDims& d, int B, const int T[3], float* base) {
  FrmScratch s;
  const long long H = d.hidden;
  float* p = base;
  auto take = [&](long long n) { float* r = p; p += n; return r; };
  for (int m = 0; m < 3; ++m) {
    const long long R = (long long)B * T[m];
    s.xw[m] = take(R * 4 * H); s.gates[m] = take(R * 4 * H); s.dgates[m] = take(R * 4 * H);
    s.cs[m] = take(R * H); s.hs[m] = take(R * H); s.hprev[m] = take(R * H);
  }
  s.hT = take(3 * B * H); s.d_hT = take(3 * B * H);
  for (int m = 0; m < 3; ++m) s.mask_h[m] = take(B * H);
  s.h3cat = take(3 * B * H); s.a1 = take(B * H); s.a2 = take(B * H); s.a3 = take(B * H);
  s.d_cat = take(3 * B * H); s.d_a1 = take(B * H); s.d_a2 = take(B * H); s.d_a3 = take(B * H);
  s.mask_cat = take(3 * B * H);
  s.d_emos = take((long long)B * d.out1); s.d_vals = take((long long)B * d.out2);
  s.d_att = take(3ll * B); s.loss_terms = take(2ll * B);
  return s;
}

int frm_check(const MerFusionDims* d, int B, const int T[3]) {
  if (int rc = check_dims(d, B)) return rc;
  MER_REQUIRE(d->hidden <= LSTM_MAXH && d->hidden % 32 == 0,
              "mer_fusion_frm: hidden %d (multiples of 32 up to %d)", d->hidden, LSTM_MAXH);
  MER_REQUIRE(T[0] > 0 && T[1] > 0 && T[2] > 0, "mer_fusion_frm: empty sequences");
  return 0;
}

// LSTM encoders + linear_1 + attention MLP (everything before the head)
int frm_forward(const MerFusionDims& d, const FrmLayout& L, const float* P, const FrmScratch& s,
                const float* const x[3], int B, const int T[3], float p_drop, const float* const masks[4],
                bool use_dropout, cudaStream_t st) {
  const int H = d.hidden;
  const int in[3] = {d.audio_dim, d.text_dim, d.video_dim};
  const float mscale = use_dropout ? 1.f / (1.f - p_drop) : 1.f;
  LinBatch lb;
  for (int m = 0; m < 3; ++m) {
    const int R = B * T[m];
    lb.p[0] = LinP{x[m], in[m], nullptr, 1.f, P + L.w_ih[m], P + L.b_ih[m], s.xw[m], 4 * H, in[m], 4 * H, 0};
    dim3 g((4 * H + 7) / 8, (R + 31) / 32, 1);
    fus_linear_fwd_kernel<<<g, 256, 0, st>>>(lb, R);
    lstm_fwd_kernel<<<B, 4 * H, 0, st>>>(s.xw[m], P + L.w_hh[m], P + L.b_hh[m], T[m], H, s.gates[m], s.cs[m],
                                         s.hs[m], s.hprev[m], s.hT + (long long)m * B * H);
  }
  for (int m = 0; m < 3; ++m)  // linear_1(dropout(h_T)), no activation, straight into the [B,3H] concat
    lb.p[m] = LinP{s.hT + (long long)m * B * H, H, use_dropout ? masks[m] : nullptr, mscale, P + L.lin_w[m],
                   P + L.lin_b[m], s.h3cat + m * H, 3 * H, H, H, 0};
  dim3 g1((H + 7) / 8, (B + 31) / 32, 3);
  fus_linear_fwd_kernel<<<g1, 256, 0, st>>>(lb, B);
  dim3 g2((H + 7) / 8, (B + 31) / 32, 1);
  lb.p[0] = LinP{s.h3cat, 3 * H, use_dropout ? masks[3] : nullptr, mscale, P + L.att_w1, P + L.att_b1, s.a1, H,
                 3 * H, H, 1};
  fus_linear_fwd_kernel<<<g2, 256, 0, st>>>(lb, B);
  lb.p[0] = LinP{s.a1, H, nullptr, 1.f, P + L.att_w2, P + L.att_b2, s.a2, H, H, H, 1};
  fus_linear_fwd_kernel<<<g2, 256, 0, st>>>(lb, B);
  lb.p[0] = LinP{s.a2, H, nullptr, 1.f, P + L.att_w3, P + L.att_b3, s.a3, H, H, H, 1};
  fus_linear_fwd_kernel<<<g2, 256, 0, st>>>(lb, B);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(10);
  return 0;
}


// ================================================================================================
// Attention_TOPN (MER2026/MER2026_Track1/toolkit/models/attention_topn.py:8-90): the utterance-level net
// generalised to N <= 18 input features, each with its own MLPEncoder; attention over the N hidden vectors.
// Same kernels as the three-modality net (three encoders per launch), a head kernel with N as a parameter.
// ================================================================================================
constexpr int TOPN_MAX = 18;

struct TopnHeadArgs {
  const float* hcat;   // [B, N*H]
  const float* a3;     // [B, H]
  const float* w_att; const float* b_att;  // [N,H],[N]
  const float* w_o1; const float* b_o1;
  const float* w_o2; const float* b_o2;
  const long long* emo; const float* val;
  float* features; float* emos_out; float* vals_out;
  float* loss_terms; float* d_emos; float* d_vals; float* d_att; float* d_cat; float* d_a3;
  int N, H, O1, O2;
  float inv_batch;
};

__global__ void __launch_bounds__(128)
fus_head_topn_kernel(const TopnHeadArgs a) {
  __shared__ float sh[4];
  __shared__ float fused[256], dfused[256];
  __shared__ float att[TOPN_MAX], datt[TOPN_MAX], logits[16], dlog[16], dval[4];
  const int b = blockIdx.x, H = a.H, N = a.N, tid = threadIdx.x;
  const float* hc = a.hcat + (long long)b * N * H;
  const float* a3 = a.a3 + (long long)b * H;
  for (int m = 0; m < N; ++m) {
    float s = 0.f;
    for (int j = tid; j < H; j += 128) s = fmaf(a.w_att[m * H + j], a3[j], s);
    s = block_sum128(s, sh);
    if (tid == 0) att[m] = s + a.b_att[m];
  }
  __syncthreads();
  for (int j = tid; j < H; j += 128) {
    float f = 0.f;
    for (int m = 0; m < N; ++m) f = fmaf(hc[m * H + j], att[m], f);
    fused[j] = f;
    a.features[(long long)b * H + j] = f;
  }
  __syncthreads();
  for (int c = 0; c < a.O1; ++c) {
    float s = 0.f;
    for (int j = tid; j < H; j += 128) s = fmaf(a.w_o1[c * H + j], fused[j], s);
    s = block_sum128(s, sh);
    if (tid == 0) { logits[c] = s + a.b_o1[c]; a.emos_out[(long long)b * a.O1 + c] = logits[c]; }
  }
  for (int c = 0; c < a.O2; ++c) {
    float s = 0.f;
    for (int j = tid; j < H; j += 128) s = fmaf(a.w_o2[c * H + j], fused[j], s);
    s = block_sum128(s, sh);
    if (tid == 0) { dval[c] = s + a.b_o2[c]; a.vals_out[(long long)b * a.O2 + c] = dval[c]; }
  }
  __syncthreads();
  if (!a.emo) return;
  if (tid == 0) {
    float mx = logits[0];
    for (int c = 1; c < a.O1; ++c) mx = fmaxf(mx, logits[c]);
    float se = 0.f;
    for (int c = 0; c < a.O1; ++c) se += expf(logits[c] - mx);
    const float lse = mx + logf(se);
    const int tgt = (int)a.emo[b];
    a.loss_terms[2 * b + 0] = lse - logits[tgt];
    for (int c = 0; c < a.O1; ++c) {
      const float sm = expf(logits[c] - lse);
      dlog[c] = (sm - (c == tgt ? 1.f : 0.f)) * a.inv_batch;
      a.d_emos[(long long)b * a.O1 + c] = dlog[c];
    }
    float mse = 0.f;
    for (int c = 0; c < a.O2; ++c) {
      const float d = dval[c] - a.val[(long long)b * a.O2 + c];
      mse += d * d;
      dval[c] = 2.f * d * a.inv_batch;
      a.d_vals[(long long)b * a.O2 + c] = dval[c];
    }
    a.loss_terms[2 * b + 1] = mse;
  }
  __syncthreads();
  for (int j = tid; j < H; j += 128) {
    float s = 0.f;
    for (int c = 0; c < a.O1; ++c) s = fmaf(a.w_o1[c * H + j], dlog[c], s);
    for (int c = 0; c < a.O2; ++c) s = fmaf(a.w_o2[c * H + j], dval[c], s);
    dfused[j] = s;
  }
  __syncthreads();
  for (int m = 0; m < N; ++m) {
    float s = 0.f;
    for (int j = tid; j < H; j += 128) s = fmaf(hc[m * H + j], dfused[j], s);
    s = block_sum128(s, sh);
    if (tid == 0) { datt[m] = s; a.d_att[(long long)N * b + m] = s; }
  }
  __syncthreads();
  for (int j = tid; j < H; j += 128) {
    float da = 0.f;
    for (int m = 0; m < N; ++m) {
      a.d_cat[(long long)b * N * H + m * H + j] = att[m] * dfused[j];
      da = fmaf(a.w_att[m * H + j], datt[m], da);
    }
    a.d_a3[(long long)b * H + j] = da;
  }
}

struct TopnLayout {
  long long enc_w1[TOPN_MAX], enc_b1[TOPN_MAX], enc_w2[TOPN_MAX], enc_b2[TOPN_MAX], enc_w3[TOPN_MAX], enc_b3[TOPN_MAX];
  long long att_w1, att_b1, att_w2, att_b2, att_w3, att_b3, fa_w, fa_b, o1_w, o1_b, o2_w, o2_b, total;
};

TopnLayout make_topn_layout(const MerFusionTopnDims& d) {
  TopnLayout L;
  long long o = 0;
  const long long H = d.hidden, N = d.n_feats;
  for (int m = 0; m < d.n_feats; ++m) {
    L.enc_w1[m] = o; o += H * d.feat_dims[m];
    L.enc_b1[m] = o; o += H;
    L.enc_w2[m] = o; o += H * H;
    L.enc_b2[m] = o; o += H;
    L.enc_w3[m] = o; o += H * H;
    L.enc_b3[m] = o; o += H;
  }
  L.att_w1 = o; o += H * N * H;
  L.att_b1 = o; o += H;
  L.att_w2 = o; o += H * H;
  L.att_b2 = o; o += H;
  L.att_w3 = o; o += H * H;
  L.att_b3 = o; o += H;
  L.fa_w = o; o += N * H;
  L.fa_b = o; o += N;
  L.o1_w = o; o += (long long)d.out1 * H;
  L.o1_b = o; o += d.out1;
  L.o2_w = o; o += (long long)d.out2 * H;
  L.o2_b = o; o += d.out2;
  L.total = o;
  return L;
}

struct TopnScratch {
  float *h1, *h2, *hcat, *a1, *a2, *a3, *d_h1, *d_h2, *d_cat, *d_a1, *d_a2, *d_a3, *d_emos, *d_vals, *d_att,
      *loss_terms, *mask_cat;
  float* mask_in[TOPN_MAX];
};

long long topn_scratch_floats(const MerFusionTopnDims& d, int B) {
  const long long H = d.hidden, N = d.n_feats;
  long long in_sum = 0;
  for (int m = 0; m < d.n_feats; ++m) in_sum += d.feat_dims[m];
  return (long long)B * (N * H * 7 + H * 6 + d.out1 + d.out2 + N + 2 + in_sum) + 64;
}

TopnScratch topn_carve(const MerFusionTopnDims& d, int B, float* base) {
  TopnScratch s;
  const long long H = d.hidden, N = d.n_feats;
  float* p = base;
  auto take = [&](long long n) { float* r = p; p += n; return r; };
  s.h1 = take(N * B * H); s.h2 = take(N * B * H); s.hcat = take(N * B * H);
  s.d_h1 = take(N * B * H); s.d_h2 = take(N * B * H); s.d_cat = take(N * B * H); s.mask_cat = take(N * B * H);
  s.a1 = take(B * H); s.a2 = take(B * H); s.a3 = take(B * H);
  s.d_a1 = take(B * H); s.d_a2 = take(B * H); s.d_a3 = take(B * H);
  s.d_emos = take((long long)B * d.out1); s.d_vals = take((long long)B * d.out2);
  s.d_att = take(N * B); s.loss_terms = take(2ll * B);
  for (int m = 0; m < d.n_feats; ++m) s.mask_in[m] = take((long long)B * d.feat_dims[m]);
  return s;
}

int topn_check(const MerFusionTopnDims* d, int B) {
  MER_REQUIRE(d && d->n_feats >= 1 && d->n_feats <= TOPN_MAX && d->hidden > 0 && d->hidden <= 256 && d->out1 > 0 &&
                  d->out1 <= 16 && d->out2 > 0 && d->out2 <= 4,
              "mer_fusion_topn: unsupported dims (1..18 features, hidden <= 256, out1 <= 16, out2 <= 4)");
  for (int m = 0; m < d->n_feats; ++m) MER_REQUIRE(d->feat_dims[m] > 0, "mer_fusion_topn: feature %d has no width", m);
  MER_REQUIRE(B > 0 && B <= 65535, "mer_fusion_topn: batch %d out of range", B);
  return 0;
}

int topn_forward(const MerFusionTopnDims& d, const TopnLayout& L, const float* P, const TopnScratch& s,
                 const float* const* x, int B, float p_drop, const float* const* masks, bool use_dropout,
                 cudaStream_t st) {
  const int H = d.hidden, N = d.n_feats;
  const float mscale = use_dropout ? 1.f / (1.f - p_drop) : 1.f;
  LinBatch lb;
  for (int m0 = 0; m0 < N; m0 += 3) {  // three encoders per launch
    const int np = min(3, N - m0);
    dim3 g1((H + 7) / 8, (B + 31) / 32, np);
    for (int i = 0; i < np; ++i) {
      const int m = m0 + i;
      lb.p[i] = LinP{x[m], d.feat_dims[m], use_dropout ? masks[m] : nullptr, mscale, P + L.enc_w1[m], P + L.enc_b1[m],
                     s.h1 + (long long)m * B * H, H, d.feat_dims[m], H, 1};
    }
    fus_linear_fwd_kernel<<<g1, 256, 0, st>>>(lb, B);
    for (int i = 0; i < np; ++i) {
      const int m = m0 + i;
      lb.p[i] = LinP{s.h1 + (long long)m * B * H, H, nullptr, 1.f, P + L.enc_w2[m], P + L.enc_b2[m],
                     s.h2 + (long long)m * B * H, H, H, H, 1};
    }
    fus_linear_fwd_kernel<<<g1, 256, 0, st>>>(lb, B);
    for (int i = 0; i < np; ++i) {
      const int m = m0 + i;
      lb.p[i] = LinP{s.h2 + (long long)m * B * H, H, nullptr, 1.f, P + L.enc_w3[m], P + L.enc_b3[m],
                     s.hcat + m * H, N * H, H, H, 1};
    }
    fus_linear_fwd_kernel<<<g1, 256, 0, st>>>(lb, B);
    mer_count_launches(3);
  }
  dim3 g2((H + 7) / 8, (B + 31) / 32, 1);
  lb.p[0] = LinP{s.hcat, N * H, use_dropout ? masks[N] : nullptr, mscale, P + L.att_w1, P + L.att_b1, s.a1, H, N * H,
                 H, 1};
  fus_linear_fwd_kernel<<<g2, 256, 0, st>>>(lb, B);
  lb.p[0] = LinP{s.a1, H, nullptr, 1.f, P + L.att_w2, P + L.att_b2, s.a2, H, H, H, 1};
  fus_linear_fwd_kernel<<<g2, 256, 0, st>>>(lb, B);
  lb.p[0] = LinP{s.a2, H, nullptr, 1.f, P + L.att_w3, P + L.att_b3, s.a3, H, H, H, 1};
  fus_linear_fwd_kernel<<<g2, 256, 0, st>>>(lb, B);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(3);
  return 0;
}

}  // namespace

extern "C" {

int mer_fusion_adam(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                    float lr, float beta1, float beta2, float eps, float weight_decay, float grad_scale,
                    float grad_clip, int* step_counter, void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(params && grads && exp_avg && exp_avg_sq && step_counter && n > 0, "mer_fusion_adam: bad operands");
  fus_adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, n, lr,
                                                              beta1, beta2, eps, weight_decay, grad_scale,
                                                              grad_clip, step_counter);
  fus_step_inc_kernel<<<1, 32, 0, st>>>(step_counter);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(2);
  return 0;
}

// ---- frame-level variant (LSTM encoders) ----------------------------------------------------------
long long mer_fusion_frm_param_count(const MerFusionDims* d) {
  if (!d) return -1;
  return make_frm_layout(*d).total;
}

long long mer_fusion_frm_workspace_bytes(const MerFusionDims* d, int max_batch, int seq_a, int seq_t, int seq_v) {
  if (!d) return -1;
  const int T[3] = {seq_a, seq_t, seq_v};
  return frm_scratch_floats(*d, max_batch, T) * 4;
}

int mer_fusion_frm_forward(const MerFusionDims* d, const float* params, const float* audios, const float* texts,
                           const float* videos, int seq_a, int seq_t, int seq_v, int B, void* workspace,
                           long long workspace_bytes, float* features, float* emos_out, float* vals_out,
                           void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const int T[3] = {seq_a, seq_t, seq_v};
  if (int rc = frm_check(d, B, T)) return rc;
  MER_REQUIRE(params && audios && texts && videos && workspace && features && emos_out && vals_out,
              "mer_fusion_frm_forward: null operand");
  MER_REQUIRE(workspace_bytes >= frm_scratch_floats(*d, B, T) * 4, "mer_fusion_frm_forward: workspace too small");
  const FrmLayout L = make_frm_layout(*d);
  const FrmScratch s = frm_carve(*d, B, T, static_cast<float*>(workspace));
  const float* x[3] = {audios, texts, videos};
  if (int rc = frm_forward(*d, L, params, s, x, B, T, 0.f, nullptr, false, st)) return rc;
  HeadArgs h;
  memset(&h, 0, sizeof(h));
  h.h3cat = s.h3cat; h.a3 = s.a3;
  h.w_att = params + L.fa_w; h.b_att = params + L.fa_b;
  h.w_o1 = params + L.o1_w; h.b_o1 = params + L.o1_b;
  h.w_o2 = params + L.o2_w; h.b_o2 = params + L.o2_b;
  h.features = features; h.emos_out = emos_out; h.vals_out = vals_out;
  h.H = d->hidden; h.O1 = d->out1; h.O2 = d->out2;
  fus_head_kernel<<<B, 128, 0, st>>>(h);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int mer_fusion_frm_fwd_bwd(const MerFusionDims* d, const float* params, float* grads, const float* audios,
                           const float* texts, const float* videos, int seq_a, int seq_t, int seq_v,
                           const int64_t* emos, const float* vals, int B, float loss_inv_batch, float dropout_p,
                           unsigned long long seed, const int* step_counter, const float* const* ext_masks,
                           void* workspace, long long workspace_bytes, float* loss_out, float* features,
                           float* emos_out, float* vals_out, void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const int T[3] = {seq_a, seq_t, seq_v};
  if (int rc = frm_check(d, B, T)) return rc;
  MER_REQUIRE(params && grads && audios && texts && videos && emos && vals && workspace && loss_out &&
                  features && emos_out && vals_out && step_counter,
              "mer_fusion_frm_fwd_bwd: null operand");
  MER_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "mer_fusion_frm_fwd_bwd: dropout %f", dropout_p);
  MER_REQUIRE(workspace_bytes >= frm_scratch_floats(*d, B, T) * 4, "mer_fusion_frm_fwd_bwd: workspace too small");
  const FrmLayout L = make_frm_layout(*d);
  const FrmScratch s = frm_carve(*d, B, T, static_cast<float*>(workspace));
  const int H = d->hidden;
  const int in[3] = {d->audio_dim, d->text_dim, d->video_dim};
  const float* x[3] = {audios, texts, videos};
  const bool drop = dropout_p > 0.f;
  const float mscale = drop ? 1.f / (1.f - dropout_p) : 1.f;
  const float* masks[4] = {nullptr, nullptr, nullptr, nullptr};
  if (drop) {
    for (int m = 0; m < 4; ++m) {  // masks 0..2 act on the [B,H] final hidden states, 3 on the concat
      if (ext_masks && ext_masks[m]) { masks[m] = ext_masks[m]; continue; }
      float* dst = m < 3 ? s.mask_h[m] : s.mask_cat;
      const long long n = (long long)B * (m < 3 ? H : 3 * H);
      fus_dropout_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
          dst, n, dropout_p, seed + 0x1000ull * (m + 1), step_counter);
      mer_count_launches(1);
      masks[m] = dst;
    }
  }
  if (int rc = frm_forward(*d, L, params, s, x, B, T, dropout_p, masks, drop, st)) return rc;
  HeadArgs h;
  memset(&h, 0, sizeof(h));
  h.h3cat = s.h3cat; h.a3 = s.a3;
  h.w_att = params + L.fa_w; h.b_att = params + L.fa_b;
  h.w_o1 = params + L.o1_w; h.b_o1 = params + L.o1_b;
  h.w_o2 = params + L.o2_w; h.b_o2 = params + L.o2_b;
  h.emo = reinterpret_cast<const long long*>(emos); h.val = vals;
  h.features = features; h.emos_out = emos_out; h.vals_out = vals_out;
  h.loss_terms = s.loss_terms; h.d_emos = s.d_emos; h.d_vals = s.d_vals; h.d_att = s.d_att;
  h.d_cat = s.d_cat; h.d_a3 = s.d_a3;
  h.H = H; h.O1 = d->out1; h.O2 = d->out2; h.inv_batch = loss_inv_batch;
  fus_head_kernel<<<B, 128, 0, st>>>(h);
  fus_loss_reduce_kernel<<<1, 32, 0, st>>>(s.loss_terms, B, loss_inv_batch, loss_out);
  mer_count_launches(2);

  float* G = grads;
  BwdBatch bb;
  auto launch_w = [&](int nprob, int K, int N, int rows) {
    dim3 g((K + 255) / 256, N, nprob);
    fus_linear_bwd_w_kernel<<<g, 256, 0, st>>>(bb, rows);
    mer_count_launches(1);
  };
  auto launch_x = [&](int nprob, int K, int rows) {
    dim3 g((K + 255) / 256, rows, nprob);
    fus_linear_bwd_x_kernel<<<g, 256, 0, st>>>(bb, rows);
    mer_count_launches(1);
  };
  bb.p[0] = BwdP{s.d_emos, d->out1, nullptr, 0, features, H, nullptr, 1.f, params + L.o1_w,
                 G + L.o1_w, G + L.o1_b, nullptr, 0, 0, H, d->out1};
  bb.p[1] = BwdP{s.d_vals, d->out2, nullptr, 0, features, H, nullptr, 1.f, params + L.o2_w,
                 G + L.o2_w, G + L.o2_b, nullptr, 0, 0, H, d->out2};
  bb.p[2] = BwdP{s.d_att, 3, nullptr, 0, s.a3, H, nullptr, 1.f, params + L.fa_w, G + L.fa_w,
                 G + L.fa_b, nullptr, 0, 0, H, 3};
  launch_w(3, H, 16, B);
  bb.p[0] = BwdP{s.d_a3, H, s.a3, H, s.a2, H, nullptr, 1.f, params + L.att_w3, G + L.att_w3,
                 G + L.att_b3, s.d_a2, H, 0, H, H};
  launch_w(1, H, H, B); launch_x(1, H, B);
  bb.p[0] = BwdP{s.d_a2, H, s.a2, H, s.a1, H, nullptr, 1.f, params + L.att_w2, G + L.att_w2,
                 G + L.att_b2, s.d_a1, H, 0, H, H};
  launch_w(1, H, H, B); launch_x(1, H, B);
  bb.p[0] = BwdP{s.d_a1, H, s.a1, H, s.h3cat, 3 * H, masks[3], mscale, params + L.att_w1,
                 G + L.att_w1, G + L.att_b1, s.d_cat, 3 * H, 1, 3 * H, H};
  launch_w(1, 3 * H, H, B); launch_x(1, 3 * H, B);
  // linear_1 of the three encoders (no activation): dW, db, and d(h_T) through the dropout mask
  for (int m = 0; m < 3; ++m)
    bb.p[m] = BwdP{s.d_cat + m * H, 3 * H, nullptr, 0, s.hT + (long long)m * B * H, H, masks[m], mscale,
                   params + L.lin_w[m], G + L.lin_w[m], G + L.lin_b[m], s.d_hT + (long long)m * B * H, H, 0, H, H};
  launch_w(3, H, H, B); launch_x(3, H, B);
  // LSTMs: BPTT per batch row, then the weight gradients as [4H, rows]^T x [rows, K] products
  for (int m = 0; m < 3; ++m) {
    const int R = B * T[m];
    lstm_bwd_kernel<<<B, 4 * H, 0, st>>>(s.d_hT + (long long)m * B * H, params + L.w_hh[m], s.gates[m], s.cs[m],
                                         T[m], H, s.dgates[m]);
    mer_count_launches(1);
    bb.p[0] = BwdP{s.dgates[m], 4 * H, nullptr, 0, x[m], in[m], nullptr, 1.f, params + L.w_ih[m], G + L.w_ih[m],
                   G + L.b_ih[m], nullptr, 0, 0, in[m], 4 * H};
    launch_w(1, in[m], 4 * H, R);
    bb.p[0] = BwdP{s.dgates[m], 4 * H, nullptr, 0, s.hprev[m], H, nullptr, 1.f, params + L.w_hh[m], G + L.w_hh[m],
                   G + L.b_hh[m], nullptr, 0, 0, H, 4 * H};
    launch_w(1, H, 4 * H, R);
  }
  MER_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// ---- Attention_TOPN (N <= 18 utterance-level features) ----------------------------------------------
long long mer_fusion_topn_param_count(const MerFusionTopnDims* d) {
  if (!d || d->n_feats < 1 || d->n_feats > TOPN_MAX) return -1;
  return make_topn_layout(*d).total;
}

long long mer_fusion_topn_workspace_bytes(const MerFusionTopnDims* d, int max_batch) {
  if (!d || d->n_feats < 1 || d->n_feats > TOPN_MAX) return -1;
  return topn_scratch_floats(*d, max_batch) * 4;
}

// feats: HOST array of n_feats device pointers, feature i is [batch, feat_dims[i]].  emos == NULL: eval-mode
// forward only (grads / loss_out / masks unused).  ext_masks: NULL or HOST array of n_feats + 1 device pointers
// (one keep-mask per input feature, then the [batch, n_feats * hidden] concat mask).
int mer_fusion_topn_step(const MerFusionTopnDims* d, const float* params, float* grads, const float* const* feats,
                         const int64_t* emos, const float* vals, int B, float loss_inv_batch, float dropout_p,
                         unsigned long long seed, const int* step_counter, const float* const* ext_masks,
                         void* workspace, long long workspace_bytes, float* loss_out, float* features,
                         float* emos_out, float* vals_out, void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (int rc = topn_check(d, B)) return rc;
  const bool train = emos != nullptr;
  MER_REQUIRE(params && feats && workspace && features && emos_out && vals_out, "mer_fusion_topn_step: null operand");
  MER_REQUIRE(!train || (grads && vals && loss_out && step_counter), "mer_fusion_topn_step: training needs grads, "
                                                                     "vals, loss_out and step_counter");
  MER_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "mer_fusion_topn_step: dropout %f", dropout_p);
  MER_REQUIRE(workspace_bytes >= topn_scratch_floats(*d, B) * 4, "mer_fusion_topn_step: workspace too small");
  const int N = d->n_feats, H = d->hidden;
  for (int m = 0; m < N; ++m) MER_REQUIRE(feats[m], "mer_fusion_topn_step: feature %d is null", m);
  const TopnLayout L = make_topn_layout(*d);
  const TopnScratch s = topn_carve(*d, B, static_cast<float*>(workspace));
  const bool drop = train && dropout_p > 0.f;
  const float mscale = drop ? 1.f / (1.f - dropout_p) : 1.f;
  const float* masks[TOPN_MAX + 1];
  for (int m = 0; m <= N; ++m) masks[m] = nullptr;
  if (drop) {
    for (int m = 0; m <= N; ++m) {
      if (ext_masks && ext_masks[m]) { masks[m] = ext_masks[m]; continue; }
      float* dst = m < N ? s.mask_in[m] : s.mask_cat;
      const long long n = (long long)B * (m < N ? d->feat_dims[m] : N * H);
      fus_dropout_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dst, n, dropout_p,
                                                                            seed + 0x1000ull * (m + 1), step_counter);
      mer_count_launches(1);
      masks[m] = dst;
    }
  }
  if (int rc = topn_forward(*d, L, params, s, feats, B, dropout_p, masks, drop, st)) return rc;
  TopnHeadArgs h;
  memset(&h, 0, sizeof(h));
  h.hcat = s.hcat; h.a3 = s.a3;
  h.w_att = params + L.fa_w; h.b_att = params + L.fa_b;
  h.w_o1 = params + L.o1_w; h.b_o1 = params + L.o1_b;
  h.w_o2 = params + L.o2_w; h.b_o2 = params + L.o2_b;
  h.features = features; h.emos_out = emos_out; h.vals_out = vals_out;
  h.N = N; h.H = H; h.O1 = d->out1; h.O2 = d->out2; h.inv_batch = loss_inv_batch;
  if (train) {
    h.emo = reinterpret_cast<const long long*>(emos); h.val = vals;
    h.loss_terms = s.loss_terms; h.d_emos = s.d_emos; h.d_vals = s.d_vals; h.d_att = s.d_att;
    h.d_cat = s.d_cat; h.d_a3 = s.d_a3;
  }
  fus_head_topn_kernel<<<B, 128, 0, st>>>(h);
  mer_count_launches(1);
  if (!train) {
    MER_CUDA_CHECK(cudaGetLastError());
    return 0;
  }
  fus_loss_reduce_kernel<<<1, 32, 0, st>>>(s.loss_terms, B, loss_inv_batch, loss_out);
  mer_count_launches(1);

  float* G = grads;
  BwdBatch bb;
  auto launch_w = [&](int nprob, int K, int Nn) {
    dim3 g((K + 255) / 256, Nn, nprob);
    fus_linear_bwd_w_kernel<<<g, 256, 0, st>>>(bb, B);
    mer_count_launches(1);
  };
  auto launch_x = [&](int nprob, int K) {
    dim3 g((K + 255) / 256, B, nprob);
    fus_linear_bwd_x_kernel<<<g, 256, 0, st>>>(bb, B);
    mer_count_launches(1);
  };
  bb.p[0] = BwdP{s.d_emos, d->out1, nullptr, 0, features, H, nullptr, 1.f, params + L.o1_w, G + L.o1_w, G + L.o1_b,
                 nullptr, 0, 0, H, d->out1};
  bb.p[1] = BwdP{s.d_vals, d->out2, nullptr, 0, features, H, nullptr, 1.f, params + L.o2_w, G + L.o2_w, G + L.o2_b,
                 nullptr, 0, 0, H, d->out2};
  bb.p[2] = BwdP{s.d_att, N, nullptr, 0, s.a3, H, nullptr, 1.f, params + L.fa_w, G + L.fa_w, G + L.fa_b, nullptr, 0, 0,
                 H, N};
  launch_w(3, H, TOPN_MAX);
  bb.p[0] = BwdP{s.d_a3, H, s.a3, H, s.a2, H, nullptr, 1.f, params + L.att_w3, G + L.att_w3, G + L.att_b3, s.d_a2, H, 0,
                 H, H};
  launch_w(1, H, H); launch_x(1, H);
  bb.p[0] = BwdP{s.d_a2, H, s.a2, H, s.a1, H, nullptr, 1.f, params + L.att_w2, G + L.att_w2, G + L.att_b2, s.d_a1, H, 0,
                 H, H};
  launch_w(1, H, H); launch_x(1, H);
  bb.p[0] = BwdP{s.d_a1, H, s.a1, H, s.hcat, N * H, masks[N], mscale, params + L.att_w1, G + L.att_w1, G + L.att_b1,
                 s.d_cat, N * H, 1, N * H, H};
  launch_w(1, N * H, H); launch_x(1, N * H);
  for (int m0 = 0; m0 < N; m0 += 3) {
    const int np = min(3, N - m0);
    for (int i = 0; i < np; ++i) {
      const int m = m0 + i;
      bb.p[i] = BwdP{s.d_cat + m * H, N * H, s.hcat + m * H, N * H, s.h2 + (long long)m * B * H, H, nullptr, 1.f,
                     params + L.enc_w3[m], G + L.enc_w3[m], G + L.enc_b3[m], s.d_h2 + (long long)m * B * H, H, 0, H, H};
    }
    launch_w(np, H, H); launch_x(np, H);
    for (int i = 0; i < np; ++i) {
      const int m = m0 + i;
      bb.p[i] = BwdP{s.d_h2 + (long long)m * B * H, H, s.h2 + (long long)m * B * H, H, s.h1 + (long long)m * B * H, H,
                     nullptr, 1.f, params + L.enc_w2[m], G + L.enc_w2[m], G + L.enc_b2[m],
                     s.d_h1 + (long long)m * B * H, H, 0, H, H};
    }
    launch_w(np, H, H); launch_x(np, H);
    int kmax = 0;
    for (int i = 0; i < np; ++i) {
      const int m = m0 + i;
      bb.p[i] = BwdP{s.d_h1 + (long long)m * B * H, H, s.h1 + (long long)m * B * H, H, feats[m], d->feat_dims[m], masks[m],
                     mscale, params + L.enc_w1[m], G + L.enc_w1[m], G + L.enc_b1[m], nullptr, 0, 0, d->feat_dims[m], H};
      kmax = d->feat_dims[m] > kmax ? d->feat_dims[m] : kmax;
    }
    launch_w(np, kmax, H);
  }
  MER_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // extern "C"
