// fusion_fused.cu — the utterance-level Attention-fusion step (MERBench/toolkit/models/attention.py:8-57 with
// MLPEncoder, modules/encoder.py:9-41; CELoss / MSELoss, toolkit/utils/loss.py:5-28; the optimiser step of
// main-release.py:50-66,205) as TWO kernels instead of one launch per layer:
//
//   fus_rows_kernel   row-parallel: a cluster of 8 CTAs owns RB batch rows and walks them through the whole
//                     network -- six dense layers forward, the attention head, both losses, and the data-gradient
//                     chain backward.  Activations of the RB rows live in shared memory, replicated in all 8
//                     CTAs; each CTA computes 1/8 of every layer's output columns (forward) or input columns
//                     (backward) and broadcasts its slice into its peers' shared memory (DSMEM), so a layer
//                     boundary costs one hardware cluster barrier, not a kernel launch or a trip through L2.
//                     Weights stream from L2 (1.9 MB at hidden 128), 1/8 of them per CTA.
//   fus_wgrad_kernel  parameter-parallel: dW[n,k] = sum_b g[b,n] x[b,k] over the whole batch for all 28 tensors in
//                     one grid, each gradient element consumed on the spot by Adam (torch.optim.Adam, coupled L2)
//                     when the step is not data-parallel; block 0 folds the per-row loss terms, the last block to
//                     finish advances the device-side step counter.
//
// fp32 SIMT throughout with a fixed summation order (no atomics on data): results are bit-reproducible, eager ==
// CUDA-graph replay.  2.86 MFLOP per clip: this is the latency regime, so the design removes launches and L2 round
// trips rather than chasing tensor cores.
#include <cooperative_groups.h>
#include <stdlib.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace cg = cooperative_groups;

namespace {

using namespace mer;

constexpr int CL = 8;      // CTAs per cluster (portable maximum)
constexpr int NT = 256;    // threads per CTA
constexpr int NW = NT / 32;
constexpr int XCH = 1024;  // staging chunk of an input row (floats)
constexpr int MAXC = 4;    // output columns per warp and layer: ceil(ceil(256 / CL) / NW)

struct ULayout {  // offsets (floats) into the flat parameter buffer, reference state_dict order
  long long enc_w1[3], enc_b1[3], enc_w2[3], enc_b2[3], enc_w3[3], enc_b3[3];
  long long att_w1, att_b1, att_w2, att_b2, att_w3, att_b3;
  long long fa_w, fa_b, o1_w, o1_b, o2_w, o2_b, total;
};

ULayout make_layout(const MerFusionDims& d) {
  ULayout L;
  long long o = 0;
  const int in[3] = {d.audio_dim, d.text_dim, d.video_dim};
  const long long H = d.hidden;
  for (int m = 0; m < 3; ++m) {
    L.enc_w1[m] = o; o += H * in[m];
    L.enc_b1[m] = o; o += H;
    L.enc_w2[m] = o; o += H * H;
    L.enc_b2[m] = o; o += H;
    L.enc_w3[m] = o; o += H * H;
    L.enc_b3[m] = o; o += H;
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

// global workspace: what the row kernel hands to the weight-gradient kernel ([B, .] row-major)
struct GWs {
  float* xd[3];               // inputs after dropout (only written / read when dropout is on)
  float *h1, *h2;             // [3][B][H] encoder activations
  float* hcd;                 // [B][3H]  concatenated encoder outputs after dropout = attention_mlp input
  float *a1, *a2, *a3;        // [B][H]
  float *g1, *g2;             // [3][B][H] gradients w.r.t. the PRE-activations of encoder layers 1, 2
  float* g3;                  // [B][3H]   same for layer 3 (concatenated layout)
  float *ga1, *ga2, *ga3;     // [B][H]    attention_mlp layers
  float *d_att, *d_emos, *d_vals, *loss_terms;  // [B][3], [B][O1], [B][O2], [B][2]
  int* done;                  // block-completion ticket of fus_wgrad_kernel
};

long long ws_floats(const MerFusionDims& d, int B) {
  const long long H = d.hidden, in_sum = (long long)d.audio_dim + d.text_dim + d.video_dim;
  return (long long)B * (in_sum + 6 * H + 3 * H + 3 * H + 6 * H + 3 * H + 3 * H + 3 + d.out1 + d.out2 + 2) + 64;
}

GWs carve(const MerFusionDims& d, int B, float* base) {
  GWs s;
  const long long H = d.hidden;
  float* p = base;
  auto take = [&](long long n) { float* r = p; p += (n + 3) / 4 * 4; return r; };  // keep 16-byte alignment
  s.done = reinterpret_cast<int*>(take(4));
  s.xd[0] = take((long long)B * d.audio_dim);
  s.xd[1] = take((long long)B * d.text_dim);
  s.xd[2] = take((long long)B * d.video_dim);
  s.h1 = take(3 * B * H); s.h2 = take(3 * B * H); s.hcd = take(3 * B * H);
  s.a1 = take(B * H); s.a2 = take(B * H); s.a3 = take(B * H);
  s.g1 = take(3 * B * H); s.g2 = take(3 * B * H); s.g3 = take(3 * B * H);
  s.ga1 = take(B * H); s.ga2 = take(B * H); s.ga3 = take(B * H);
  s.d_att = take(3ll * B); s.d_emos = take((long long)B * d.out1); s.d_vals = take((long long)B * d.out2);
  s.loss_terms = take(2ll * B);
  return s;
}

enum { MODE_FWD = 0, MODE_LOSS = 1, MODE_UPSTREAM = 2, MODE_FWD_TRAIN = 3 };  // eval forward | fused loss step | backward from upstream gradients | train-mode forward only

struct RowArgs {
  MerFusionDims d;
  ULayout L;
  const float* P;
  const float* x[3];
  const float* ext_mask[4];            // device keep-masks (0/1) or null -> counter hash
  const long long* emo; const float* val;                     // MODE_LOSS
  const float *up_feat, *up_emos, *up_vals;                   // MODE_UPSTREAM (each may be null)
  int B, mode;
  float inv_batch, p_drop, mscale;
  unsigned long long seed;
  const int* step;
  float *features, *emos_out, *vals_out;
  GWs ws;
};

// the keep-mask of fusion.cu:fus_dropout_mask_kernel, element i of mask tensor m
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

__device__ __forceinline__ float warp_allsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float dot4(const float4& a, const float4& b, float acc) {
  acc = fmaf(a.x, b.x, acc);
  acc = fmaf(a.y, b.y, acc);
  acc = fmaf(a.z, b.z, acc);
  return fmaf(a.w, b.w, acc);
}

// acc[c][r] += sum_k in[r][k] * W[n_c][k] over k in [0, K) for this warp's columns n_c = n0 + warp + NW c < n1;
// `in` is shared memory [RB][ldin]; lanes stride over k (float4 when rows are 16-byte aligned).
template <int RB>
__device__ __forceinline__ void accumulate_cols(float (&acc)[MAXC][RB], const float* __restrict__ in, int ldin, int K,
                                                const float* __restrict__ W, long long ldw, int n0, int n1) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool vec = (K % 4 == 0) && (ldw % 4 == 0) && (ldin % 4 == 0) && ((reinterpret_cast<size_t>(W) & 15) == 0);
  if (vec) {
#pragma unroll 3
    for (int k4 = lane; k4 < K / 4; k4 += 32) {
      float4 w[MAXC];
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        const int n = n0 + warp + NW * c;
        if (n < n1) w[c] = __ldg(reinterpret_cast<const float4*>(W + (long long)n * ldw) + k4);
      }
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        const float4 xv = *reinterpret_cast<const float4*>(in + r * ldin + 4 * k4);
#pragma unroll
        for (int c = 0; c < MAXC; ++c)
          if (n0 + warp + NW * c < n1) acc[c][r] = dot4(xv, w[c], acc[c][r]);
      }
    }
  } else {
    for (int k = lane; k < K; k += 32) {
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        const int n = n0 + warp + NW * c;
        if (n >= n1) continue;
        const float w = __ldg(W + (long long)n * ldw + k);
#pragma unroll
        for (int r = 0; r < RB; ++r) acc[c][r] = fmaf(in[r * ldin + k], w, acc[c][r]);
      }
    }
  }
}

// Finish this warp's columns: cross-lane sum, then emit(c, n, r, value) on every lane (all lanes hold the sums).
template <int RB, class Emit>
__device__ __forceinline__ void finish_cols(float (&acc)[MAXC][RB], int n0, int n1, Emit emit) {
  const int warp = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int n = n0 + warp + NW * c;
    if (n >= n1) continue;
#pragma unroll
    for (int r = 0; r < RB; ++r) emit(n, r, warp_allsum(acc[c][r]));
  }
}

// dx[r][k] = sum_n dy[r][n] W[n][k] for this CTA's input columns k in [k0, k1): thread = (k, n-lane), partial sums
// over n-lanes meet in `red`, then fin(r, k, sum).  dy: shared [RB][lddy].
template <int RB, class Fin>
__device__ __forceinline__ void backward_cols(const float* __restrict__ dy, int lddy, int N, const float* __restrict__ W,
                                              long long ldw, int k0, int k1, float* red, Fin fin) {
  const int KS = k1 - k0;
  if (KS > 0) {
    const int NL = NT / KS;  // KS <= 96: at least two n-lanes
    const int tid = threadIdx.x;
    if (tid < KS * NL) {
      const int kk = tid % KS, nl = tid / KS;
      float acc[RB];
#pragma unroll
      for (int r = 0; r < RB; ++r) acc[r] = 0.f;
#pragma unroll 8
      for (int n = nl; n < N; n += NL) {
        const float w = __ldg(W + (long long)n * ldw + k0 + kk);
#pragma unroll
        for (int r = 0; r < RB; ++r) acc[r] = fmaf(dy[r * lddy + n], w, acc[r]);
      }
#pragma unroll
      for (int r = 0; r < RB; ++r) red[(nl * RB + r) * KS + kk] = acc[r];
    }
    __syncthreads();
    for (int i = tid; i < RB * KS; i += NT) {
      const int r = i / KS, kk = i % KS;
      float s = 0.f;
      for (int nl = 0; nl < NL; ++nl) s += red[(nl * RB + r) * KS + kk];
      fin(r, k0 + kk, s);
    }
  } else {
    __syncthreads();
  }
  __syncthreads();
}

// The attention head of Attention.forward (attention.py:44-53) for the RB rows of a cluster, replicated in every CTA
// (warp r <-> row r: no exchange needed): att = fc_att(a3), fused = [h_a h_t h_v] att, the two output heads, and --
// when a backward pass follows -- the loss terms / upstream gradients, d fused, the head's share of d(concat) (g3h)
// and the gradient w.r.t. the pre-activation of attention_mlp.linear_3 (ga3).  All buffers are shared memory.
// JM: elements of a hidden vector per lane (hidden <= 32 JM); MO1: emotion classes the unrolled code covers.  The fast
// kernel instantiates <4, 4, 8>: this code runs ONCE per launch, straight from a cold instruction cache, so its size is
// its cost (the <4, 8, 16> form is 2.5x as long).
template <int RB, int JM = 8, int MO1 = 16>
__device__ __forceinline__ void head_rows(const RowArgs& a, int rank, int row0, bool train, const float* hc,
                                          const float* a3, float* feat, float* dfu, float* g3h, float* ga3,
                                          const float* head_w = nullptr, long long* tr = nullptr) {
#define HEAD_TR(i)                                                                        \
  do {                                                                                    \
    if (tr != nullptr && blockIdx.x == 0 && threadIdx.x == 0) tr[i] = clock64();          \
  } while (0)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int H = a.d.hidden, H3 = 3 * H, B = a.B, O1 = a.d.out1, O2 = a.d.out2;
  // the head's parameters (fc_att, fc_out_1, fc_out_2: contiguous from L.fa_w to L.total) read from global memory, or
  // from a copy the caller has put in shared memory (head_w[i] = P[L.fa_w + i])
  // Parameter tensors of the head, as pointers into global memory or into the caller's shared-memory copy
  const float* Wb = head_w ? head_w : a.P + a.L.fa_w;   // Wb[i] = P[L.fa_w + i]
  const float* w_att = Wb;
  const float* b_att = Wb + (a.L.fa_b - a.L.fa_w);
  const float* w_o1 = Wb + (a.L.o1_w - a.L.fa_w);
  const float* b_o1 = Wb + (a.L.o1_b - a.L.fa_w);
  const float* w_o2 = Wb + (a.L.o2_w - a.L.fa_w);
  const float* b_o2 = Wb + (a.L.o2_b - a.L.fa_w);
  // One warp per row, and every stage written so that its independent pieces are in flight together (the first build
  // ran ten dot products one after the other on a scheduler with no other warp to hide their latencies: ~1k cycles each)
  for (int r = warp; r < RB; r += NW) {
    const int row = row0 + r;
    const bool live = row < B;
    const float* a3r = a3 + r * H;
    const float* hcr = hc + r * H3;
    float att[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < JM; ++i) {
      const int j = lane + 32 * i;
      if (j < H) {
        const float x = a3r[j];
#pragma unroll
        for (int m = 0; m < 3; ++m) att[m] = fmaf(w_att[m * H + j], x, att[m]);
      }
    }
#pragma unroll
    for (int m = 0; m < 3; ++m) att[m] = warp_allsum(att[m]) + b_att[m];
    HEAD_TR(0);
    float f[JM];
    float logit[MO1], vout[4];
#pragma unroll
    for (int c = 0; c < MO1; ++c) logit[c] = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) vout[c] = 0.f;
#pragma unroll
    for (int i = 0; i < JM; ++i) {
      const int j = lane + 32 * i;
      f[i] = 0.f;
      if (j < H) {
        f[i] = (hcr[j] * att[0] + hcr[H + j] * att[1]) + hcr[2 * H + j] * att[2];
        feat[r * H + j] = f[i];
        if (rank == 0 && live) a.features[(long long)row * H + j] = f[i];
#pragma unroll
        for (int c = 0; c < MO1; ++c)
          if (c < O1) logit[c] = fmaf(w_o1[c * H + j], f[i], logit[c]);
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < O2) vout[c] = fmaf(w_o2[c * H + j], f[i], vout[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < MO1; ++c)
      if (c < O1) logit[c] = warp_allsum(logit[c]) + b_o1[c];
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (c < O2) vout[c] = warp_allsum(vout[c]) + b_o2[c];
    if (rank == 0 && live && lane == 0) {
#pragma unroll
      for (int c = 0; c < MO1; ++c)
        if (c < O1) a.emos_out[(long long)row * O1 + c] = logit[c];
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < O2) a.vals_out[(long long)row * O2 + c] = vout[c];
    }
    HEAD_TR(1);
    if (!train) continue;
    // upstream gradients of the two heads (every lane computes the same scalars)
    float dlog[MO1], dval[4];
#pragma unroll
    for (int c = 0; c < MO1; ++c) dlog[c] = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) dval[c] = 0.f;
    if (a.mode == MODE_LOSS) {
      // CELoss: NLL(log_softmax) summed / N; MSELoss: squared error summed / N  (loss.py:11-28)
      const int tgt = live ? (int)a.emo[row] : 0;   // (issued first: the loads fly while the softmax is evaluated)
      float tval[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) tval[c] = (live && c < O2) ? a.val[(long long)row * O2 + c] : 0.f;
      float mx = logit[0];
#pragma unroll
      for (int c = 1; c < MO1; ++c)
        if (c < O1) mx = fmaxf(mx, logit[c]);
      float se = 0.f;
#pragma unroll
      for (int c = 0; c < MO1; ++c)
        if (c < O1) se += expf(logit[c] - mx);
      const float lse = mx + logf(se);
      float ce = 0.f, mse = 0.f;
#pragma unroll
      for (int c = 0; c < MO1; ++c) {
        if (c < O1) {
          if (c == tgt) ce = lse - logit[c];
          dlog[c] = live ? (expf(logit[c] - lse) - (c == tgt ? 1.f : 0.f)) * a.inv_batch : 0.f;
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (c < O2) {
          const float dd = live ? vout[c] - tval[c] : 0.f;
          mse += dd * dd;
          dval[c] = 2.f * dd * a.inv_batch;
        }
      }
      if (rank == 0 && live && lane == 0) {
        a.ws.loss_terms[2 * row] = ce;
        a.ws.loss_terms[2 * row + 1] = mse;
      }
    } else {
#pragma unroll
      for (int c = 0; c < MO1; ++c)
        if (c < O1) dlog[c] = (live && a.up_emos) ? a.up_emos[(long long)row * O1 + c] : 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < O2) dval[c] = (live && a.up_vals) ? a.up_vals[(long long)row * O2 + c] : 0.f;
    }
    if (rank == 0 && live && lane == 0) {
#pragma unroll
      for (int c = 0; c < MO1; ++c)
        if (c < O1) a.ws.d_emos[(long long)row * O1 + c] = dlog[c];
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < O2) a.ws.d_vals[(long long)row * O2 + c] = dval[c];
    }
    HEAD_TR(2);
    float datt[3] = {0.f, 0.f, 0.f};
    float df[JM];
#pragma unroll
    for (int i = 0; i < JM; ++i) {
      const int j = lane + 32 * i;
      df[i] = 0.f;
      if (j < H) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < MO1; ++c)
          if (c < O1) s = fmaf(w_o1[c * H + j], dlog[c], s);
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < O2) s = fmaf(w_o2[c * H + j], dval[c], s);
        if (a.mode == MODE_UPSTREAM && a.up_feat && live) s += a.up_feat[(long long)row * H + j];
        df[i] = s;
        dfu[r * H + j] = s;
#pragma unroll
        for (int m = 0; m < 3; ++m) datt[m] = fmaf(hcr[m * H + j], s, datt[m]);
      }
    }
#pragma unroll
    for (int m = 0; m < 3; ++m) datt[m] = warp_allsum(datt[m]);
    HEAD_TR(3);
    if (rank == 0 && live && lane < 3) a.ws.d_att[3 * row + lane] = lane == 0 ? datt[0] : (lane == 1 ? datt[1] : datt[2]);
#pragma unroll
    for (int i = 0; i < JM; ++i) {
      const int j = lane + 32 * i;
      if (j < H) {
        const float s = df[i];
#pragma unroll
        for (int m = 0; m < 3; ++m) g3h[r * H3 + m * H + j] = att[m] * s;
        const float da3 = (w_att[j] * datt[0] + w_att[H + j] * datt[1]) + w_att[2 * H + j] * datt[2];
        const float g = a3r[j] > 0.f ? da3 : 0.f;
        ga3[r * H + j] = g;
        if (rank == 0 && live) a.ws.ga3[(long long)row * H + j] = g;
      }
    }
  }
}

template <int RB>
__global__ void __launch_bounds__(NT, 1) fus_rows_kernel(const __grid_constant__ RowArgs a) {
  extern __shared__ __align__(16) float smem[];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = a.d.hidden, H3 = 3 * H, B = a.B;
  const int O1 = a.d.out1, O2 = a.d.out2;
  const int in[3] = {a.d.audio_dim, a.d.text_dim, a.d.video_dim};
  const int row0 = (int)(blockIdx.x / CL) * RB;
  const bool drop = a.p_drop > 0.f && a.mode != MODE_FWD;
  const bool train = a.mode == MODE_LOSS || a.mode == MODE_UPSTREAM;  // backward follows: keep what it needs
  const int step = drop ? *a.step : 0;
  const float* P = a.P;

  // ---- shared-memory carve (identical in every CTA of the cluster: peers are addressed by the same offsets) ----
  float* sp = smem;
  auto take = [&](int n) { float* r = sp; sp += n; return r; };
  float* xs = take(RB * XCH);
  float* h1 = take(3 * RB * H);   // [m][r][H]
  float* h2 = take(3 * RB * H);
  float* hc = take(RB * H3);      // [r][3H] encoder outputs (before dropout)
  float* hcd = take(RB * H3);     // after dropout
  float* mf = take(RB * H3);      // dropout factor (mask * scale) of the concat
  float* a1 = take(RB * H);
  float* a2 = take(RB * H);
  float* a3 = take(RB * H);
  float* feat = take(RB * H);
  float* dfu = take(RB * H);      // d loss / d fused features
  float* g3h = take(RB * H3);     // head's contribution to d(concat)
  float* g3p = take(RB * H3);     // gradient w.r.t. the pre-activation of encoder layer 3
  float* ga1 = take(RB * H);
  float* ga2 = take(RB * H);
  float* ga3 = take(RB * H);
  float* g2 = take(3 * RB * H);
  float* red = take(NT * RB);

  const int HC = (H + CL - 1) / CL;
  const int n0 = min(H, rank * HC), n1 = min(H, n0 + HC);          // this CTA's slice of an H-wide layer
  const int C3 = (H3 + CL - 1) / CL;
  const int c0 = min(H3, rank * C3), c1 = min(H3, c0 + C3);        // ... of the 3H-wide concat

  if (blockIdx.x == 0 && tid == 0 && train) *a.ws.done = 0;
  cluster.sync();  // every CTA of the cluster is running: DSMEM stores may begin

  // all 8 peers' views of a local shared buffer (lanes 0..7 each keep one)
  auto peer = [&](float* local) { return cluster.map_shared_rank(local, lane & (CL - 1)); };

  // ================= forward =================
  // encoder layer 1: inputs come from global memory in chunks (dropout applied while staging)
  for (int m = 0; m < 3; ++m) {
    const int K = in[m];
    const float* W = P + a.L.enc_w1[m];
    float acc[MAXC][RB];
#pragma unroll
    for (int c = 0; c < MAXC; ++c)
#pragma unroll
      for (int r = 0; r < RB; ++r) acc[c][r] = 0.f;
    for (int k0 = 0, chunk = 0; k0 < K; k0 += XCH, ++chunk) {
      const int kc = min(XCH, K - k0);
      const bool writer = drop && train && rank == (m + chunk) % CL;
      for (int r = 0; r < RB; ++r) {
        const int row = row0 + r;
        for (int k = tid; k < kc; k += NT) {
          float v = 0.f;
          if (row < B) {
            const long long i = (long long)row * K + k0 + k;
            v = a.x[m][i];
            if (drop) {
              const float keep = a.ext_mask[m] ? a.ext_mask[m][i] : keep_hash(a.seed, m, step, i, a.p_drop);
              v *= keep * a.mscale;
              if (writer) a.ws.xd[m][i] = v;
            }
          }
          xs[r * XCH + k] = v;
        }
      }
      __syncthreads();
      accumulate_cols<RB>(acc, xs, XCH, kc, W + k0, K, n0, n1);
      __syncthreads();
    }
    float* dst = peer(h1);
    finish_cols<RB>(acc, n0, n1, [&](int n, int r, float v) {
      v = fmaxf(v + P[a.L.enc_b1[m] + n], 0.f);
      if (lane < CL) dst[(m * RB + r) * H + n] = v;
      if (lane == CL + r && train && row0 + r < B) a.ws.h1[((long long)m * B + row0 + r) * H + n] = v;
    });
  }
  cluster.sync();
  // encoder layer 2
  for (int m = 0; m < 3; ++m) {
    float acc[MAXC][RB] = {};
    accumulate_cols<RB>(acc, h1 + m * RB * H, H, H, P + a.L.enc_w2[m], H, n0, n1);
    float* dst = peer(h2);
    finish_cols<RB>(acc, n0, n1, [&](int n, int r, float v) {
      v = fmaxf(v + P[a.L.enc_b2[m] + n], 0.f);
      if (lane < CL) dst[(m * RB + r) * H + n] = v;
      if (lane == CL + r && train && row0 + r < B) a.ws.h2[((long long)m * B + row0 + r) * H + n] = v;
    });
  }
  cluster.sync();
  // encoder layer 3 -> concat (+ dropout of the concat)
  for (int m = 0; m < 3; ++m) {
    float acc[MAXC][RB] = {};
    accumulate_cols<RB>(acc, h2 + m * RB * H, H, H, P + a.L.enc_w3[m], H, n0, n1);
    float* dhc = peer(hc);
    float* dhcd = peer(hcd);
    float* dmf = peer(mf);
    finish_cols<RB>(acc, n0, n1, [&](int n, int r, float v) {
      v = fmaxf(v + P[a.L.enc_b3[m] + n], 0.f);
      const int row = row0 + r, col = m * H + n;
      float f = 1.f;
      if (drop && row < B) {
        const long long i = (long long)row * H3 + col;
        f = (a.ext_mask[3] ? a.ext_mask[3][i] : keep_hash(a.seed, 3, step, i, a.p_drop)) * a.mscale;
      }
      if (lane < CL) {
        dhc[r * H3 + col] = v;
        dhcd[r * H3 + col] = v * f;
        dmf[r * H3 + col] = f;
      }
      if (lane == CL + r && train && row < B) a.ws.hcd[(long long)row * H3 + col] = v * f;
    });
  }
  cluster.sync();
  // attention_mlp
  {
    float acc[MAXC][RB] = {};
    accumulate_cols<RB>(acc, hcd, H3, H3, P + a.L.att_w1, H3, n0, n1);
    float* dst = peer(a1);
    finish_cols<RB>(acc, n0, n1, [&](int n, int r, float v) {
      v = fmaxf(v + P[a.L.att_b1 + n], 0.f);
      if (lane < CL) dst[r * H + n] = v;
      if (lane == CL + r && train && row0 + r < B) a.ws.a1[(long long)(row0 + r) * H + n] = v;
    });
  }
  cluster.sync();
  {
    float acc[MAXC][RB] = {};
    accumulate_cols<RB>(acc, a1, H, H, P + a.L.att_w2, H, n0, n1);
    float* dst = peer(a2);
    finish_cols<RB>(acc, n0, n1, [&](int n, int r, float v) {
      v = fmaxf(v + P[a.L.att_b2 + n], 0.f);
      if (lane < CL) dst[r * H + n] = v;
      if (lane == CL + r && train && row0 + r < B) a.ws.a2[(long long)(row0 + r) * H + n] = v;
    });
  }
  cluster.sync();
  {
    float acc[MAXC][RB] = {};
    accumulate_cols<RB>(acc, a2, H, H, P + a.L.att_w3, H, n0, n1);
    float* dst = peer(a3);
    finish_cols<RB>(acc, n0, n1, [&](int n, int r, float v) {
      v = fmaxf(v + P[a.L.att_b3 + n], 0.f);
      if (lane < CL) dst[r * H + n] = v;
      if (lane == CL + r && train && row0 + r < B) a.ws.a3[(long long)(row0 + r) * H + n] = v;
    });
  }
  cluster.sync();

  // ================= head (replicated in every CTA) =================
  head_rows<RB>(a, rank, row0, train, hc, a3, feat, dfu, g3h, ga3);
  if (!train) {
    cluster.sync();  // no CTA may exit while a peer could still be storing into its shared memory
    return;
  }
  __syncthreads();

  // ================= backward: data gradients =================
  // attention_mlp.linear_3 -> d a2 (every finisher broadcasts its value into the 8 copies of the buffer)
  backward_cols<RB>(ga3, H, H, P + a.L.att_w3, H, n0, n1, red, [&](int r, int k, float s) {
    const float g = a2[r * H + k] > 0.f ? s : 0.f;
    for (int p = 0; p < CL; ++p) cluster.map_shared_rank(ga2, p)[r * H + k] = g;
    if (row0 + r < B) a.ws.ga2[(long long)(row0 + r) * H + k] = g;
  });
  cluster.sync();
  backward_cols<RB>(ga2, H, H, P + a.L.att_w2, H, n0, n1, red, [&](int r, int k, float s) {
    const float g = a1[r * H + k] > 0.f ? s : 0.f;
    for (int p = 0; p < CL; ++p) cluster.map_shared_rank(ga1, p)[r * H + k] = g;
    if (row0 + r < B) a.ws.ga1[(long long)(row0 + r) * H + k] = g;
  });
  cluster.sync();
  // attention_mlp.linear_1 -> d concat (through the concat dropout), plus the head's share, through layer 3's ReLU
  backward_cols<RB>(ga1, H, H, P + a.L.att_w1, H3, c0, c1, red, [&](int r, int k, float s) {
    const float tot = g3h[r * H3 + k] + s * mf[r * H3 + k];
    const float g = hc[r * H3 + k] > 0.f ? tot : 0.f;
    for (int p = 0; p < CL; ++p) cluster.map_shared_rank(g3p, p)[r * H3 + k] = g;
    if (row0 + r < B) a.ws.g3[(long long)(row0 + r) * H3 + k] = g;
  });
  cluster.sync();
  for (int m = 0; m < 3; ++m) {  // encoder layer 3 -> d h2
    backward_cols<RB>(g3p + m * H, H3, H, P + a.L.enc_w3[m], H, n0, n1, red, [&](int r, int k, float s) {
      const float g = h2[(m * RB + r) * H + k] > 0.f ? s : 0.f;
      for (int p = 0; p < CL; ++p) cluster.map_shared_rank(g2, p)[(m * RB + r) * H + k] = g;
      if (row0 + r < B) a.ws.g2[((long long)m * B + row0 + r) * H + k] = g;
    });
  }
  cluster.sync();
  for (int m = 0; m < 3; ++m) {  // encoder layer 2 -> d h1 (the input gradient of layer 1 is not needed)
    backward_cols<RB>(g2 + m * RB * H, H, H, P + a.L.enc_w2[m], H, n0, n1, red, [&](int r, int k, float s) {
      const float g = h1[(m * RB + r) * H + k] > 0.f ? s : 0.f;
      if (row0 + r < B) a.ws.g1[((long long)m * B + row0 + r) * H + k] = g;
    });
  }
  // the last DSMEM stores (g2) were fenced by the barrier above: CTAs may retire independently
}

// ---------------------------------------------------------------------------------------------------------------
// fus_rows_fast_kernel — the same row-parallel pass for the common shapes (hidden <= 128, feature widths that are
// multiples of 4 and fit the plan below), rebuilt around what the first version measured: per step at
// B = 32, almost all of it exposed L2 latency (every layer began with a dependent weight load) -- not arithmetic.
//   * Weights come in through the bulk-copy engine (cp.async.bulk + mbarrier), never through a load a warp waits on:
//     this CTA's row slices W[n0:n1, :] of the five hidden-layer matrices (88 KB at hidden 128) are requested at kernel
//     entry and stay in shared memory for BOTH directions; layer 1's slices (the bulk of the bytes) stream through two
//     chunk buffers while the previous chunk is being consumed.
//   * The backward pass splits the SAME row slices: CTA c holds rows n0:n1 of W and the gradient of exactly those
//     pre-activations (it produced them), so it computes the partial d x[r, :] over its 16 n's for every input column
//     and scatters the column slices to their owners through DSMEM (a reduce-scatter; 8 partials summed in rank
//     order -> deterministic).  No weight is read twice, no gradient is broadcast.
//   * 12 cluster barriers per step (6 forward layers, 5 backward exchanges, 1 at entry), each ~0.3 us of hardware.
long long* g_fus_trace = nullptr;  // debug: clock64 stamps of block 0 / thread 0 (scripts/micro/fusion_trace.py)
constexpr int FRB = 4;        // rows per cluster
constexpr int HCP = 16;       // slice width bound: ceil(128 / 8)
constexpr int FMAXC = 2;      // columns per warp: ceil(16 / 8)

struct FastPlan {             // shared-memory offsets (floats) + sizes, computed on the host, identical in every CTA
  int xs[3];                  // [FRB][in_m] staged inputs (after dropout)
  int h1, h2, hc, hcd, a1, a2, a3, feat, dfu, g3h, ga3;   // activations / head gradients (full copies)
  int own_a, own_3, own_2;    // this CTA's slices of pre-activation gradients: [FRB][HCP], [3][FRB][HCP] x 2
  int rx;                     // [2][CL][3][FRB][HCP] reduce-scatter landing zones (ping-pong)
  int wb;                     // [3][rch][max_in] layer-1 weight chunks: rch whole rows of W1[m] = ONE bulk copy each
  int t2, t3, ta1, ta2, ta3;  // resident row slices
  int hw;                     // head parameters fc_att | fc_out_1 | fc_out_2 (weights and biases)
  int sl;                     // [2][3][FRB][HCP] this CTA's freshly computed output slices, before they are broadcast
  int bars;                   // 4 mbarriers (2 chunk buffers, resident set, spare)
  int rch, max_in;            // layer-1 chunk: rows per chunk, row pitch of the buffers
  int total;                  // floats
};

FastPlan make_fast_plan(const MerFusionDims& d, int rch) {
  FastPlan p;
  const int H = d.hidden;
  const int in[3] = {d.audio_dim, d.text_dim, d.video_dim};
  int o = 0;
  auto take = [&](int n) { int r = o; o += (n + 3) & ~3; return r; };
  for (int m = 0; m < 3; ++m) p.xs[m] = take(FRB * in[m]);
  p.h1 = take(3 * FRB * H);
  // everything written after layer 1 (by this CTA or by its peers, who have passed the same cluster barrier) may live
  // where the staged inputs were: they are dead by then
  const int xs_end = o;
  const bool alias = 17 * FRB * H <= xs_end - p.xs[0] - 3 * FRB * H - 16;
  if (alias) o = p.xs[0];
  p.h2 = take(3 * FRB * H);
  p.hc = take(FRB * 3 * H); p.hcd = take(FRB * 3 * H);
  p.a1 = take(FRB * H); p.a2 = take(FRB * H); p.a3 = take(FRB * H);
  p.feat = take(FRB * H); p.dfu = take(FRB * H);
  p.g3h = take(FRB * 3 * H);
  if (alias) o = xs_end;
  p.ga3 = take(FRB * H);
  p.own_a = take(FRB * HCP); p.own_3 = take(3 * FRB * HCP); p.own_2 = take(3 * FRB * HCP);
  p.max_in = in[0] > in[1] ? (in[0] > in[2] ? in[0] : in[2]) : (in[1] > in[2] ? in[1] : in[2]);
  p.rch = rch;
  p.wb = take(3 * rch * p.max_in);      // three chunk buffers: two copies in flight behind the one being consumed
  p.rx = p.wb;                          // the landing zones of the backward exchanges reuse them (layer 1 is long done)
  if (3 * rch * p.max_in < 2 * CL * 3 * FRB * HCP) take(2 * CL * 3 * FRB * HCP - 3 * rch * p.max_in);
  p.t2 = take(3 * HCP * H); p.t3 = take(3 * HCP * H);
  p.ta1 = take(HCP * 3 * H); p.ta2 = take(HCP * H); p.ta3 = take(HCP * H);
  p.hw = take(3 * H + 3 + (d.out1 + d.out2) * (H + 1));
  p.sl = take(2 * 3 * FRB * HCP);
  p.bars = take(8);
  p.total = o;
  return p;
}

__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
                   "r"(smem_u32(dst_smem)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// acc[c][r] += sum_k in[r][k] * tile[c_local][k]: `tile` is a shared-memory row slice [nloc][ldt]
__device__ __forceinline__ void fast_accumulate(float (&acc)[FMAXC][FRB], const float* __restrict__ in, int ldin, int K,
                                                const float* __restrict__ tile, int ldt, int nloc) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k4 = lane; k4 < K / 4; k4 += 32) {
    float4 w[FMAXC];
#pragma unroll
    for (int c = 0; c < FMAXC; ++c)
      if (warp + NW * c < nloc) w[c] = *reinterpret_cast<const float4*>(tile + (warp + NW * c) * ldt + 4 * k4);
#pragma unroll
    for (int r = 0; r < FRB; ++r) {
      const float4 xv = *reinterpret_cast<const float4*>(in + r * ldin + 4 * k4);
#pragma unroll
      for (int c = 0; c < FMAXC; ++c)
        if (warp + NW * c < nloc) acc[c][r] = dot4(xv, w[c], acc[c][r]);
    }
  }
}

template <class Emit>
__device__ __forceinline__ void fast_finish(float (&acc)[FMAXC][FRB], int n0, int nloc, Emit emit) {
  const int warp = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < FMAXC; ++c) {
    if (warp + NW * c >= nloc) continue;
#pragma unroll
    for (int r = 0; r < FRB; ++r) emit(n0 + warp + NW * c, r, warp_allsum(acc[c][r]));
  }
}

__global__ void __launch_bounds__(NT, 1) fus_rows_fast_kernel(const __grid_constant__ RowArgs a,
                                                              const __grid_constant__ FastPlan pl,
                                                              long long* __restrict__ trace) {
#define FUS_TR(slot)                                                                  \
  do {                                                                                \
    if (trace != nullptr && blockIdx.x == 0 && threadIdx.x == 0) trace[slot] = clock64(); \
  } while (0)
  FUS_TR(0);
  extern __shared__ __align__(16) float smem[];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = a.d.hidden, H3 = 3 * H, B = a.B;
  const int in[3] = {a.d.audio_dim, a.d.text_dim, a.d.video_dim};
  const int row0 = (int)(blockIdx.x / CL) * FRB;
  const bool drop = a.p_drop > 0.f && a.mode != MODE_FWD;
  const bool train = a.mode == MODE_LOSS || a.mode == MODE_UPSTREAM;
  const int step = drop ? *a.step : 0;
  const float* P = a.P;
  const int HC = (H + CL - 1) / CL;
  const int n0 = min(H, rank * HC), n1 = min(H, n0 + HC), nloc = n1 - n0;

  float* xs[3] = {smem + pl.xs[0], smem + pl.xs[1], smem + pl.xs[2]};
  float* h1 = smem + pl.h1; float* h2 = smem + pl.h2; float* hc = smem + pl.hc; float* hcd = smem + pl.hcd;
  float* a1 = smem + pl.a1; float* a2 = smem + pl.a2; float* a3 = smem + pl.a3;
  float* feat = smem + pl.feat; float* dfu = smem + pl.dfu; float* g3h = smem + pl.g3h; float* ga3 = smem + pl.ga3;
  float* own_a = smem + pl.own_a; float* own_3 = smem + pl.own_3; float* own_2 = smem + pl.own_2;
  float* rx = smem + pl.rx; float* wb = smem + pl.wb;
  float* t2 = smem + pl.t2; float* t3 = smem + pl.t3; float* ta1 = smem + pl.ta1; float* ta2 = smem + pl.ta2;
  float* ta3 = smem + pl.ta3;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + pl.bars);  // [0..2]: chunk buffers; [3]: resident tiles

  float* hw = smem + pl.hw;
  float* sl = smem + pl.sl;
  const int rch = pl.rch, wb_ld = pl.max_in;
  // layer-1 chunk list: modality m, rows [n0 + rch c, + rch) of W1[m] (whole rows: contiguous in the parameter buffer,
  // ONE bulk copy per chunk -- the first build issued one copy per row and spent 29k cycles here, ~200 per copy)
  const int cpm = (nloc + rch - 1) / rch;  // chunks per modality
  const int nc_total = 3 * cpm;
  auto issue_chunk = [&](int c) {  // one thread
    const int m = c / cpm, r0 = (c % cpm) * rch, rows = min(rch, nloc - r0);
    uint64_t* bar = &bars[c % 3];
    const uint32_t bytes = (uint32_t)(rows * in[m] * 4);
    mbar_expect_tx(bar, bytes);
    bulk_g2s(wb + (c % 3) * rch * wb_ld, P + a.L.enc_w1[m] + (long long)(n0 + r0) * in[m], bytes, bar);
  };

  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    mbar_init(&bars[2], 1);
    mbar_init(&bars[3], 1);   // resident tiles
    fence_mbar_init();
    if (blockIdx.x == 0 && train) *a.ws.done = 0;
    mbar_expect_tx(&bars[3], (uint32_t)(nloc * (6 * H + 3 * H + 2 * H) * 4));
  }
  __syncthreads();
  // the copies are issued by eight different warps (one thread issuing all twelve held its warp -- and with it the
  // whole CTA at the next barrier -- for ~10k cycles)
  if (lane == 0 && nloc > 0) {
    if (warp < 3 && warp < nc_total) issue_chunk(warp);
    if (warp >= 3 && warp < 6) {
      const int m = warp - 3;
      bulk_g2s(t2 + m * HCP * H, P + a.L.enc_w2[m] + (long long)n0 * H, (uint32_t)(nloc * H * 4), &bars[3]);
      bulk_g2s(t3 + m * HCP * H, P + a.L.enc_w3[m] + (long long)n0 * H, (uint32_t)(nloc * H * 4), &bars[3]);
    }
    if (warp == 6) bulk_g2s(ta1, P + a.L.att_w1 + (long long)n0 * H3, (uint32_t)(nloc * H3 * 4), &bars[3]);
    if (warp == 7) {
      bulk_g2s(ta2, P + a.L.att_w2 + (long long)n0 * H, (uint32_t)(nloc * H * 4), &bars[3]);
      bulk_g2s(ta3, P + a.L.att_w3 + (long long)n0 * H, (uint32_t)(nloc * H * 4), &bars[3]);
    }
  }
  // the head's parameters and the three inputs of the FRB rows: plain copies first (independent 16-byte loads, many in
  // flight per thread -- the first build hashed element by element behind each dependent load: 26k cycles), dropout
  // applied in place afterwards by the thread that copied the element
  {
    const int n_hw = (int)(a.L.total - a.L.fa_w);
    for (int i = tid; i < n_hw; i += NT) hw[i] = P[a.L.fa_w + i];
    for (int m = 0; m < 3; ++m) {
      const int K4 = in[m] >> 2;
      const float4* src = reinterpret_cast<const float4*>(a.x[m]) + (long long)row0 * K4;
      float4* dst = reinterpret_cast<float4*>(xs[m]);
      const int live4 = max(0, min(FRB, B - row0)) * K4;
#pragma unroll 4
      for (int i = tid; i < FRB * K4; i += NT) dst[i] = i < live4 ? src[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (drop) {
      for (int m = 0; m < 3; ++m) {
        const int K = in[m];
        const int live = max(0, min(FRB, B - row0)) * K;
        for (int i4 = tid; i4 < (FRB * K) >> 2; i4 += NT) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int i = 4 * i4 + e;
            if (i < live) {
              const long long gi = (long long)row0 * K + i;
              const float v = xs[m][i] * (a.ext_mask[m] ? a.ext_mask[m][gi] : keep_hash(a.seed, m, step, gi, a.p_drop)) * a.mscale;
              xs[m][i] = v;
              if (train && rank == m) a.ws.xd[m][gi] = v;
            }
          }
        }
      }
    }
  }
  __syncthreads();
  FUS_TR(1);
  cluster.sync();  // every CTA of the cluster is running: DSMEM stores may begin
  FUS_TR(2);

  // Totals of a warp's 2 x 4 partial sums with 9 shuffles instead of 40: halves are exchanged, not duplicated; lane l
  // ends up with the total of (column slot c = bit 4 of l, row r = bits 3..2 of l); lanes with l % 4 == 0 use it.
  auto reduce_2x4 = [&](float (&acc)[FMAXC][FRB]) {
    float v[8];
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
      for (int r = 0; r < 4; ++r) v[c * 4 + r] = acc[c][r];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float keep = (lane & 16) ? v[i + 4] : v[i], send = (lane & 16) ? v[i] : v[i + 4];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float keep = (lane & 8) ? v[i + 2] : v[i], send = (lane & 8) ? v[i] : v[i + 2];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
    {
      const float keep = (lane & 4) ? v[1] : v[0], send = (lane & 4) ? v[0] : v[1];
      v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 2);
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
    return v[0];
  };
  // this warp's finished outputs -> the CTA's slice buffer sl[which][m][r][nl] (value = relu(total + bias))
  auto to_slice = [&](float (&acc)[FMAXC][FRB], int which, int m, const float* bias, auto post) {
    const float tot = reduce_2x4(acc);
    if ((lane & 3) == 0) {
      const int c = lane >> 4, r = (lane >> 2) & 3, nl = warp + NW * c;
      if (nl < nloc) post(which, m, r, nl, fmaxf(tot + bias[n0 + nl], 0.f));
    }
  };
  // slice buffer -> the eight copies of the activation buffer (16-byte DSMEM stores, one or two per thread) and, when a
  // backward pass follows, global memory for the weight-gradient kernel
  auto broadcast = [&](int which, int nmod, float* act, int act_ld_row, int act_mod_stride, float* gdst, long long g_mod_stride,
                       int g_ld) {
    __syncthreads();
    const int f4n = nloc >> 2;
    for (int i = tid; i < nmod * FRB * f4n * CL; i += NT) {
      const int peer_rank = i % CL, q = i / CL;
      const int f4 = q % f4n, r = (q / f4n) % FRB, m = q / (f4n * FRB);
      const float4 v4 = *reinterpret_cast<const float4*>(sl + ((which * 3 + m) * FRB + r) * HCP + 4 * f4);
      float* dst = cluster.map_shared_rank(act, peer_rank);
      *reinterpret_cast<float4*>(dst + m * act_mod_stride + r * act_ld_row + n0 + 4 * f4) = v4;
    }
    if (train && gdst != nullptr) {
      for (int q = tid; q < nmod * FRB * f4n; q += NT) {
        const int f4 = q % f4n, r = (q / f4n) % FRB, m = q / (f4n * FRB);
        if (row0 + r < B)
          *reinterpret_cast<float4*>(gdst + m * g_mod_stride + (long long)(row0 + r) * g_ld + n0 + 4 * f4) =
              *reinterpret_cast<const float4*>(sl + ((which * 3 + m) * FRB + r) * HCP + 4 * f4);
      }
    }
  };
  auto plain = [&](int which, int m, int r, int nl, float v) { sl[((which * 3 + m) * FRB + r) * HCP + nl] = v; };

  // ================= forward =================
  {
    float acc[FMAXC][FRB] = {};
    for (int c = 0; c < nc_total; ++c) {
      const int m = c / cpm, r0 = (c % cpm) * rch, rows = min(rch, nloc - r0);
      mbar_wait(&bars[c % 3], (c / 3) & 1);
      // this chunk's `rows` columns: warp w takes local columns r0 + w, r0 + w + 8 (accumulator slot = chunk parity when
      // a chunk holds up to 8 rows, so that the 2 x 4 totals of a modality are reduced together)
      {
        const float* tile = wb + (c % 3) * rch * wb_ld;
        const int K4 = in[m] >> 2;
        for (int k4 = lane; k4 < K4; k4 += 32) {
#pragma unroll
          for (int cc = 0; cc < FMAXC; ++cc) {
            const int rl = warp + NW * cc;       // row inside the chunk
            const int slot = (r0 + rl) / NW;     // accumulator slot of local column r0 + rl (= warp + NW * slot)
            if (rl < rows && slot < FMAXC) {
              const float4 w4 = *reinterpret_cast<const float4*>(tile + rl * in[m] + 4 * k4);
#pragma unroll
              for (int r = 0; r < FRB; ++r) {
                const float4 xv = *reinterpret_cast<const float4*>(xs[m] + r * in[m] + 4 * k4);
                if (slot == 0) acc[0][r] = dot4(xv, w4, acc[0][r]);
                else acc[1][r] = dot4(xv, w4, acc[1][r]);
              }
            }
          }
        }
      }
      __syncthreads();  // every warp is done with this buffer
      if (tid == 0 && c + 3 < nc_total) issue_chunk(c + 3);
      if ((c + 1) % cpm == 0) {  // last chunk of modality m: its layer-1 output
        to_slice(acc, 0, m, P + a.L.enc_b1[m], plain);
#pragma unroll
        for (int ci = 0; ci < FMAXC; ++ci)
#pragma unroll
          for (int r = 0; r < FRB; ++r) acc[ci][r] = 0.f;
      }
    }
  }
  FUS_TR(3);
  broadcast(0, 3, h1, H, FRB * H, a.ws.h1, (long long)B * H, H);
  cluster.sync();
  FUS_TR(4);
  mbar_wait(&bars[3], 0);  // resident tiles (requested at entry: long since there)
  FUS_TR(5);
  auto cat_factor = [&](int row, int col) {  // dropout factor of concat element (row, col)
    if (!drop || row >= B) return 1.f;
    const long long gi = (long long)row * H3 + col;
    return (a.ext_mask[3] ? a.ext_mask[3][gi] : keep_hash(a.seed, 3, step, gi, a.p_drop)) * a.mscale;
  };
  // The five hidden layers behind layer 1, ONE copy of the code in a loop over a small table: this kernel executes every
  // instruction once per launch out of a cold instruction cache, so code size IS time (the unrolled first build spent
  // ~8 cycles per SASS instruction; halving the head's code halved its time).
#pragma unroll 1
  for (int L = 0; L < 5; ++L) {
    const float *inb, *tileb;
    float* act;
    float* gdst;
    long long bias0 = 0, g_ms = 0;
    int nmod = 1, ldin = H, K = H, in_ms = 0, tile_ms = 0, act_ms = 0, act_ld = H, g_ld = H;
    if (L == 0) {         // encoder layer 2
      inb = h1; tileb = t2; act = h2; gdst = a.ws.h2;
      nmod = 3; in_ms = FRB * H; tile_ms = HCP * H; act_ms = FRB * H; g_ms = (long long)B * H;
    } else if (L == 1) {  // encoder layer 3 -> concat (slice 0: as computed, slice 1: after the concat's dropout)
      inb = h2; tileb = t3; act = hc; gdst = nullptr;
      nmod = 3; in_ms = FRB * H; tile_ms = HCP * H; act_ms = H; act_ld = H3;
    } else if (L == 2) {  // attention_mlp
      inb = hcd; tileb = ta1; act = a1; gdst = a.ws.a1; bias0 = a.L.att_b1; ldin = H3; K = H3;
    } else if (L == 3) {
      inb = a1; tileb = ta2; act = a2; gdst = a.ws.a2; bias0 = a.L.att_b2;
    } else {
      inb = a2; tileb = ta3; act = a3; gdst = a.ws.a3; bias0 = a.L.att_b3;
    }
#pragma unroll 1
    for (int m = 0; m < nmod; ++m) {
      float acc[FMAXC][FRB] = {};
      fast_accumulate(acc, inb + m * in_ms, ldin, K, tileb + m * tile_ms, K, nloc);
      const long long boff = L == 0 ? a.L.enc_b2[m] : (L == 1 ? a.L.enc_b3[m] : bias0);
      to_slice(acc, 0, m, P + boff, [&](int, int mm, int r, int nl, float v) {
        sl[((0 * 3 + mm) * FRB + r) * HCP + nl] = v;
        if (L == 1) sl[((1 * 3 + mm) * FRB + r) * HCP + nl] = v * cat_factor(row0 + r, mm * H + n0 + nl);
      });
    }
    broadcast(0, nmod, act, act_ld, act_ms, gdst, g_ms, g_ld);
    if (L == 1) broadcast(1, 3, hcd, H3, H, a.ws.hcd, H, H3);
    cluster.sync();
  }
  FUS_TR(9);

  head_rows<FRB, 4, 8>(a, rank, row0, train, hc, a3, feat, dfu, g3h, ga3, hw, trace ? trace + 16 : nullptr);
  FUS_TR(10);
  if (!train) {
    cluster.sync();
    FUS_TR(11);
    return;
  }
  __syncthreads();

  // ================= backward: reduce-scatter of partial data gradients (five exchanges, one copy of the code) ========
  // own slice of the head's gradient w.r.t. attention_mlp.linear_3's pre-activation
  for (int i = tid; i < FRB * nloc; i += NT) own_a[(i / nloc) * HCP + i % nloc] = ga3[(i / nloc) * H + n0 + i % nloc];
#pragma unroll 1
  for (int e = 0; e < 5; ++e) {
    // exchange e: this CTA's pre-activation gradients `down` (slots of [FRB][HCP]) times its row slices `tileb` give
    // partial input gradients for all K columns; column j of slot s goes to CTA j / HC; the owner adds the 8 partials in
    // rank order, applies the ReLU mask of the activation it belongs to, keeps the result as its own `down` for the next
    // exchange and writes it to global memory for the weight-gradient kernel.
    const float *down, *tileb, *relu_act;
    float *own_dst, *gdst;
    int nsrc = 1, K = H, tile_ms = 0, nslot = 1, act_ss = 0, act_rs = H;
    long long g_ss = 0, g_rs = H;
    const int zone = e & 1;
    if (e == 0) {         // attention_mlp.linear_3 -> d a2
      down = own_a; tileb = ta3; relu_act = a2; own_dst = own_a; gdst = a.ws.ga2;
    } else if (e == 1) {  // linear_2 -> d a1
      down = own_a; tileb = ta2; relu_act = a1; own_dst = own_a; gdst = a.ws.ga1;
    } else if (e == 2) {  // linear_1 -> d concat (slot = modality), plus the head's share, through the concat dropout
      down = own_a; tileb = ta1; K = H3; nslot = 3; relu_act = hc; act_ss = H; act_rs = H3; own_dst = own_3; gdst = a.ws.g3;
      g_ss = H; g_rs = H3;
    } else if (e == 3) {  // encoder layer 3 -> d h2
      down = own_3; tileb = t3; nsrc = 3; tile_ms = HCP * H; nslot = 3; relu_act = h2; act_ss = FRB * H; own_dst = own_2;
      gdst = a.ws.g2; g_ss = (long long)B * H;
    } else {              // encoder layer 2 -> d h1 (the input gradient of layer 1 is not needed)
      down = own_2; tileb = t2; nsrc = 3; tile_ms = HCP * H; nslot = 3; relu_act = h1; act_ss = FRB * H; own_dst = nullptr;
      gdst = a.ws.g1; g_ss = (long long)B * H;
    }
    __syncthreads();
    float* zbase = rx + zone * (CL * 3 * FRB * HCP);
#pragma unroll 1
    for (int src = 0; src < nsrc; ++src) {
      const float* dn = down + src * FRB * HCP;
      const float* tl = tileb + src * tile_ms;
      for (int k = tid; k < K; k += NT) {
        float acc[FRB] = {0.f, 0.f, 0.f, 0.f};
        for (int nl = 0; nl < nloc; ++nl) {
          const float w = tl[nl * K + k];
#pragma unroll
          for (int r = 0; r < FRB; ++r) acc[r] = fmaf(dn[r * HCP + nl], w, acc[r]);
        }
        const int slot = src + k / H, j = k % H;
        const int dest = j / HC, kk = j - dest * HC;
        float* z = cluster.map_shared_rank(zbase, dest);
#pragma unroll
        for (int r = 0; r < FRB; ++r) z[((rank * 3 + slot) * FRB + r) * HCP + kk] = acc[r];
      }
    }
    if (e == 0) FUS_TR(11);
    cluster.sync();
    if (e == 0) FUS_TR(12);
    for (int i = tid; i < nslot * FRB * nloc; i += NT) {
      const int kk = i % nloc, r = (i / nloc) % FRB, slot = i / (nloc * FRB);
      float v = 0.f;
#pragma unroll
      for (int src = 0; src < CL; ++src) v += zbase[((src * 3 + slot) * FRB + r) * HCP + kk];
      const int k = n0 + kk;
      if (e == 2) v = g3h[r * H3 + slot * H + k] + v * cat_factor(row0 + r, slot * H + k);
      const float g = relu_act[slot * act_ss + r * act_rs + k] > 0.f ? v : 0.f;
      if (own_dst != nullptr) own_dst[(slot * FRB + r) * HCP + kk] = g;
      if (row0 + r < B) gdst[slot * g_ss + (long long)(row0 + r) * g_rs + k] = g;
    }
  }
  FUS_TR(13);
  // zone 0 was last written before the barrier above and zone 1 two barriers ago: CTAs may retire independently
}

// ---------------------------------------------------------------------------------------------------------------
struct WProb {
  const float* dy; int lddy;
  const float* x; int ldx;
  int N, K;
  long long w_off, b_off;
  int blk0;
};
struct WArgs {
  WProb p[15];
  int nblocks, B;
  float* G;
  float *P, *M, *V;     // Adam operands (do_adam)
  float lr, beta1, beta2, eps, wd, clip;
  int do_adam;
  int* step;
  int* done;
  const float* loss_terms; float inv_batch; float* loss_out;
};

// torch.optim.Adam (coupled L2), same operation order as fusion.cu:fus_adam_kernel; bc1 / bc2_sqrt are the bias
// corrections 1 - beta1^t and sqrt(1 - beta2^t) of this step (computed once per thread)
__device__ __forceinline__ void adam_update(const WArgs& a, long long i, float grad, float bc1, float bc2_sqrt) {
  if (a.clip > 0.f) grad = fminf(fmaxf(grad, -a.clip), a.clip);
  float mi = a.M[i], vi = a.V[i];
  a.P[i] = mer::adam_param(a.P[i], grad, mi, vi, a.lr, a.beta1, a.beta2, a.eps, a.wd, bc1, bc2_sqrt);
  a.M[i] = mi;
  a.V[i] = vi;
}

// VW outputs dW[n, k .. k + VW) per thread (VW = 4 when every K is a multiple of 4 and the activations are 16-byte
// aligned: one 16-byte load of x per batch row instead of four scalar ones -- the kernel is load-issue bound; per
// element the sum over the batch runs in the same order in both forms, so they agree bit for bit)
template <int VW>
__global__ void __launch_bounds__(NT) fus_wgrad_kernel(const __grid_constant__ WArgs a) {
  const int tid = threadIdx.x;
  float bc1 = 1.f, bc2_sqrt = 1.f;
  if (a.do_adam) {
    const float t = (float)(*a.step + 1);
    bc1 = 1.f - powf(a.beta1, t);
    bc2_sqrt = sqrtf(1.f - powf(a.beta2, t));
  }
  int pi = 0;
#pragma unroll
  for (int i = 1; i < 15; ++i)
    if ((int)blockIdx.x >= a.p[i].blk0) pi = i;
  const WProb& p = a.p[pi];
  const long long e = ((long long)(blockIdx.x - p.blk0) * NT + tid) * VW;
  if (e < (long long)p.N * p.K) {
    const int n = (int)(e / p.K), k = (int)(e % p.K);  // K % VW == 0: the VW outputs share n
    float acc[VW] = {}, accb = 0.f;
    const float* dy = p.dy + n;
    const float* x = p.x + k;
#pragma unroll 8
    for (int b = 0; b < a.B; ++b) {
      const float g = dy[(long long)b * p.lddy];
      accb += g;
      if (VW == 4) {
        const float4 xv = *reinterpret_cast<const float4*>(x + (long long)b * p.ldx);
        acc[0] = fmaf(g, xv.x, acc[0]);
        acc[1 % VW] = fmaf(g, xv.y, acc[1 % VW]);
        acc[2 % VW] = fmaf(g, xv.z, acc[2 % VW]);
        acc[3 % VW] = fmaf(g, xv.w, acc[3 % VW]);
      } else {
        acc[0] = fmaf(g, x[(long long)b * p.ldx], acc[0]);
      }
    }
#pragma unroll
    for (int j = 0; j < VW; ++j) {
      a.G[p.w_off + e + j] = acc[j];
      if (a.do_adam) adam_update(a, p.w_off + e + j, acc[j], bc1, bc2_sqrt);
    }
    if (k == 0) {
      a.G[p.b_off + n] = accb;
      if (a.do_adam) adam_update(a, p.b_off + n, accb, bc1, bc2_sqrt);
    }
  }
  if (blockIdx.x == 0 && tid == 0 && a.loss_out) {
    float ce = 0.f, mse = 0.f;
    for (int b = 0; b < a.B; ++b) { ce += a.loss_terms[2 * b]; mse += a.loss_terms[2 * b + 1]; }
    a.loss_out[0] = ce * a.inv_batch;
    a.loss_out[1] = mse * a.inv_batch;
    a.loss_out[2] = ce * a.inv_batch + mse * a.inv_batch;
  }
  if (a.do_adam) {  // the last block to get here advances the step counter (every block has read it by then)
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      if (atomicAdd(a.done, 1) == (int)gridDim.x - 1) {
        *a.step = *a.step + 1;
        *a.done = 0;
      }
    }
  }
}

int check_dims(const MerFusionDims* d, int B) {
  MER_REQUIRE(d && d->hidden >= 4 && d->hidden <= 256 && d->hidden % 4 == 0 && d->out1 > 0 && d->out1 <= 16 &&
                  d->out2 > 0 && d->out2 <= 4 && d->audio_dim > 0 && d->text_dim > 0 && d->video_dim > 0,
              "mer_fusion: unsupported dims (hidden a multiple of 4 up to 256, out1 <= 16, out2 <= 4)");
  MER_REQUIRE(B > 0 && B <= 65535, "mer_fusion: batch %d out of range", B);
  return 0;
}

size_t rows_smem_bytes(int H, int RB) { return sizeof(float) * (size_t)RB * (XCH + 32 * (size_t)H + NT); }

template <int RB>
int launch_rows_t(const RowArgs& a, cudaStream_t st) {
  static MerPerDevice once;
  const size_t smem = rows_smem_bytes(a.d.hidden, RB);
  if (once.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(fus_rows_kernel<RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    once.mark();
  }
  MER_REQUIRE(smem <= 200 * 1024, "mer_fusion: shared-memory plan of %zu bytes", smem);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(CL * ((a.B + RB - 1) / RB)));
  cfg.blockDim = dim3(NT);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  MER_CUDA_CHECK(cudaLaunchKernelEx(&cfg, fus_rows_kernel<RB>, a));
  mer_count_launches(1);
  return 0;
}

// fast path: hidden <= 128 (a multiple of 4), feature widths multiples of 4, everything within 227 KB of shared memory
bool fast_plan_for(const MerFusionDims& d, FastPlan* out) {
  const int in[3] = {d.audio_dim, d.text_dim, d.video_dim};
  if (d.hidden > 128 || d.hidden % 32 != 0 || d.out1 > 8) return false;  // slices of hidden / 8 columns move as 16-byte vectors
  for (int m = 0; m < 3; ++m)
    if (in[m] % 4 != 0) return false;
  // layer-1 chunks hold 8 whole rows of W1[m] (one per warp: the accumulator slots rely on it)
  const FastPlan p = make_fast_plan(d, 8);
  if ((size_t)p.total * 4 <= 227 * 1024) {
    *out = p;
    return true;
  }
  return false;
}

int launch_rows_fast(const RowArgs& a, const FastPlan& pl, cudaStream_t st) {
  static MerPerDevice once;
  if (once.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(fus_rows_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    once.mark();
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(CL * ((a.B + FRB - 1) / FRB)));
  cfg.blockDim = dim3(NT);
  cfg.dynamicSmemBytes = (size_t)pl.total * 4;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  MER_CUDA_CHECK(cudaLaunchKernelEx(&cfg, fus_rows_fast_kernel, a, pl, g_fus_trace));
  mer_count_launches(1);
  return 0;
}

int launch_rows(const RowArgs& a, cudaStream_t st) {
  static const bool no_fast = getenv("MER_FUSION_GENERIC") != nullptr;  // A/B and fallback testing
  // the fast kernel stages the input rows with 16-byte loads (its widths are multiples of 4, so every row is aligned
  // when the base pointer is); a caller's view that starts off a 16-byte boundary takes the general kernel
  bool aligned = true;
  for (int m = 0; m < 3; ++m) aligned = aligned && (reinterpret_cast<uintptr_t>(a.x[m]) & 15) == 0;
  FastPlan pl;
  if (!no_fast && aligned && fast_plan_for(a.d, &pl)) return launch_rows_fast(a, pl, st);
  // 8 rows per cluster once there are enough rows to fill the GPU with clusters and the plan fits shared memory
  if (a.B >= 128 && a.d.hidden <= 128) return launch_rows_t<8>(a, st);
  return launch_rows_t<4>(a, st);
}

int launch_wgrad(const MerFusionDims& d, const ULayout& L, const GWs& ws, const float* const x[3], bool drop, int B,
                 float* grads, const float* features, float* params, float* exp_avg, float* exp_avg_sq,
                 const MerAdamHyper* adam, int* step, float inv_batch, float* loss_out, cudaStream_t st) {
  WArgs w;
  memset(&w, 0, sizeof(w));
  const int H = d.hidden;
  const int in[3] = {d.audio_dim, d.text_dim, d.video_dim};
  int np = 0, blk = 0;
  // four outputs per thread when every K is a multiple of 4 and every activation row starts on a 16-byte boundary
  // (the workspace buffers do by construction; the inputs and `features` are the caller's)
  bool vec = in[0] % 4 == 0 && in[1] % 4 == 0 && in[2] % 4 == 0 && (reinterpret_cast<uintptr_t>(features) & 15) == 0;
  for (int m = 0; m < 3; ++m) vec = vec && (reinterpret_cast<uintptr_t>(drop ? ws.xd[m] : x[m]) & 15) == 0;
  static const bool no_vec = getenv("MER_FUSION_WGRAD_SCALAR") != nullptr;  // A/B and bit-equality tests
  if (no_vec) vec = false;
  const int per_block = NT * (vec ? 4 : 1);
  auto add = [&](const float* dy, int lddy, const float* xin, int ldx, int N, int K, long long w_off, long long b_off) {
    w.p[np] = WProb{dy, lddy, xin, ldx, N, K, w_off, b_off, blk};
    blk += (int)(((long long)N * K + per_block - 1) / per_block);
    ++np;
  };
  for (int m = 0; m < 3; ++m) {
    add(ws.g1 + (long long)m * B * H, H, drop ? ws.xd[m] : x[m], in[m], H, in[m], L.enc_w1[m], L.enc_b1[m]);
    add(ws.g2 + (long long)m * B * H, H, ws.h1 + (long long)m * B * H, H, H, H, L.enc_w2[m], L.enc_b2[m]);
    add(ws.g3 + m * H, 3 * H, ws.h2 + (long long)m * B * H, H, H, H, L.enc_w3[m], L.enc_b3[m]);
  }
  add(ws.ga1, H, ws.hcd, 3 * H, H, 3 * H, L.att_w1, L.att_b1);
  add(ws.ga2, H, ws.a1, H, H, H, L.att_w2, L.att_b2);
  add(ws.ga3, H, ws.a2, H, H, H, L.att_w3, L.att_b3);
  add(ws.d_att, 3, ws.a3, H, 3, H, L.fa_w, L.fa_b);
  add(ws.d_emos, d.out1, features, H, d.out1, H, L.o1_w, L.o1_b);
  add(ws.d_vals, d.out2, features, H, d.out2, H, L.o2_w, L.o2_b);
  w.nblocks = blk;
  w.B = B;
  w.G = grads;
  if (adam) {
    w.do_adam = 1;
    w.P = params; w.M = exp_avg; w.V = exp_avg_sq;
    w.lr = adam->lr; w.beta1 = adam->beta1; w.beta2 = adam->beta2; w.eps = adam->eps;
    w.wd = adam->weight_decay; w.clip = adam->grad_clip;
  }
  w.step = step;
  w.done = ws.done;
  w.loss_terms = ws.loss_terms;
  w.inv_batch = inv_batch;
  w.loss_out = loss_out;
  if (vec) fus_wgrad_kernel<4><<<blk, NT, 0, st>>>(w);
  else fus_wgrad_kernel<1><<<blk, NT, 0, st>>>(w);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

int fill_rows(RowArgs& a, const MerFusionDims* d, const float* params, const float* audios, const float* texts,
              const float* videos, int B, float dropout_p, unsigned long long seed, const int* step,
              const float* const* ext_masks, void* workspace, long long workspace_bytes, float* features,
              float* emos_out, float* vals_out) {
  if (int rc = check_dims(d, B)) return rc;
  MER_REQUIRE(params && audios && texts && videos && workspace && features && emos_out && vals_out,
              "mer_fusion: null operand");
  MER_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "mer_fusion: dropout %f", dropout_p);
  MER_REQUIRE(dropout_p == 0.f || step, "mer_fusion: dropout needs the step counter");
  MER_REQUIRE(workspace_bytes >= ws_floats(*d, B) * 4, "mer_fusion: workspace too small");
  memset(&a, 0, sizeof(a));
  a.d = *d;
  a.L = make_layout(*d);
  a.P = params;
  a.x[0] = audios; a.x[1] = texts; a.x[2] = videos;
  if (ext_masks)
    for (int m = 0; m < 4; ++m) a.ext_mask[m] = ext_masks[m];
  a.B = B;
  a.p_drop = dropout_p;
  a.mscale = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
  a.seed = seed;
  a.step = step;
  a.features = features; a.emos_out = emos_out; a.vals_out = vals_out;
  a.ws = carve(*d, B, static_cast<float*>(workspace));
  return 0;
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) void mer_debug_fusion_trace(long long* device_buffer) { g_fus_trace = device_buffer; }

long long mer_fusion_param_count(const MerFusionDims* d) {
  if (!d) return -1;
  return make_layout(*d).total;
}

long long mer_fusion_workspace_bytes(const MerFusionDims* d, int max_batch) {
  if (!d) return -1;
  return ws_floats(*d, max_batch) * 4;
}

int mer_fusion_forward(const MerFusionDims* d, const float* params, const float* audios, const float* texts,
                       const float* videos, int B, void* workspace, long long workspace_bytes, float* features,
                       float* emos_out, float* vals_out, void* stream_) {
  RowArgs a;
  if (int rc = fill_rows(a, d, params, audios, texts, videos, B, 0.f, 0, nullptr, nullptr, workspace, workspace_bytes,
                         features, emos_out, vals_out))
    return rc;
  a.mode = MODE_FWD;
  return launch_rows(a, static_cast<cudaStream_t>(stream_));
}

int mer_fusion_fwd_bwd(const MerFusionDims* d, const float* params, float* grads, const float* audios,
                       const float* texts, const float* videos, const int64_t* emos, const float* vals, int B,
                       float loss_inv_batch, float dropout_p, unsigned long long seed, const int* step_counter,
                       const float* const* ext_masks, void* workspace, long long workspace_bytes, float* loss_out,
                       float* features, float* emos_out, float* vals_out, void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  RowArgs a;
  if (int rc = fill_rows(a, d, params, audios, texts, videos, B, dropout_p, seed, step_counter, ext_masks, workspace,
                         workspace_bytes, features, emos_out, vals_out))
    return rc;
  MER_REQUIRE(grads && emos && vals && loss_out && step_counter, "mer_fusion_fwd_bwd: null operand");
  a.mode = MODE_LOSS;
  a.emo = reinterpret_cast<const long long*>(emos);
  a.val = vals;
  a.inv_batch = loss_inv_batch;
  if (int rc = launch_rows(a, st)) return rc;
  return launch_wgrad(*d, a.L, a.ws, a.x, dropout_p > 0.f, B, grads, features, nullptr, nullptr, nullptr, nullptr,
                      nullptr, loss_inv_batch, loss_out, st);
}

int mer_fusion_step(const MerFusionDims* d, float* params, float* grads, float* exp_avg, float* exp_avg_sq,
                    const float* audios, const float* texts, const float* videos, const int64_t* emos,
                    const float* vals, int B, float loss_inv_batch, float dropout_p, unsigned long long seed,
                    int* step_counter, const float* const* ext_masks, const MerAdamHyper* adam, void* workspace,
                    long long workspace_bytes, float* loss_out, float* features, float* emos_out, float* vals_out,
                    void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  RowArgs a;
  if (int rc = fill_rows(a, d, params, audios, texts, videos, B, dropout_p, seed, step_counter, ext_masks, workspace,
                         workspace_bytes, features, emos_out, vals_out))
    return rc;
  MER_REQUIRE(grads && exp_avg && exp_avg_sq && emos && vals && loss_out && step_counter && adam,
              "mer_fusion_step: null operand");
  a.mode = MODE_LOSS;
  a.emo = reinterpret_cast<const long long*>(emos);
  a.val = vals;
  a.inv_batch = loss_inv_batch;
  if (int rc = launch_rows(a, st)) return rc;
  return launch_wgrad(*d, a.L, a.ws, a.x, dropout_p > 0.f, B, grads, features, params, exp_avg, exp_avg_sq, adam,
                      step_counter, loss_inv_batch, loss_out, st);
}

int mer_fusion_forward_train(const MerFusionDims* d, const float* params, const float* audios, const float* texts,
                             const float* videos, int B, float dropout_p, unsigned long long seed,
                             const int* step_counter, const float* const* ext_masks, void* workspace,
                             long long workspace_bytes, float* features, float* emos_out, float* vals_out,
                             void* stream_) {
  RowArgs a;
  if (int rc = fill_rows(a, d, params, audios, texts, videos, B, dropout_p, seed, step_counter, ext_masks, workspace,
                         workspace_bytes, features, emos_out, vals_out))
    return rc;
  a.mode = MODE_FWD_TRAIN;
  return launch_rows(a, static_cast<cudaStream_t>(stream_));
}

int mer_fusion_backward(const MerFusionDims* d, const float* params, float* grads, const float* audios,
                        const float* texts, const float* videos, int B, const float* d_features,
                        const float* d_emos, const float* d_vals, float dropout_p, unsigned long long seed,
                        const int* step_counter, const float* const* ext_masks, void* workspace,
                        long long workspace_bytes, float* features, float* emos_out, float* vals_out, void* stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  RowArgs a;
  if (int rc = fill_rows(a, d, params, audios, texts, videos, B, dropout_p, seed, step_counter, ext_masks, workspace,
                         workspace_bytes, features, emos_out, vals_out))
    return rc;
  MER_REQUIRE(grads, "mer_fusion_backward: null operand");
  a.mode = MODE_UPSTREAM;
  a.up_feat = d_features; a.up_emos = d_emos; a.up_vals = d_vals;
  if (int rc = launch_rows(a, st)) return rc;
  return launch_wgrad(*d, a.L, a.ws, a.x, dropout_p > 0.f, B, grads, features, nullptr, nullptr, nullptr, nullptr,
                      nullptr, 0.f, nullptr, st);
}

}  // extern "C"
