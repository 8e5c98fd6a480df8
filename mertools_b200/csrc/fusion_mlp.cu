// fusion_mlp.cu — the MER2023 challenge baseline nets (MER2023/main-release.py:226-290, MLP and Attention with a free
// `--layers` list), their loss (CELoss + MSELoss, :293-315) and one optimisation step (:363-369), table-driven for chains
// of 1..8 layers of width 1..1024 and input widths of any size:
//
//   mlp_rows_kernel   row-parallel: a cluster of 8 CTAs owns RB batch rows and walks them through every chain
//                     (Linear -> ReLU -> Dropout per layer), the head, both losses and the data-gradient chain back.
//                     The rows' current activations live in shared memory, replicated in all 8 CTAs; each CTA computes
//                     1/8 of a layer's output columns (forward) or input columns (backward) and stores its slice into
//                     its peers' shared memory (DSMEM), so a layer boundary costs one cluster barrier.  What the
//                     weight gradients need (each layer's output and pre-activation gradient) goes to the workspace.
//   mlp_wgrad_kernel  parameter-parallel: dW[n,k] = sum_b g[b,n] x[b,k] for every tensor of the net in one grid, in a
//                     fixed order over the batch; block 0 folds the per-row loss terms.
//
// The Adam update is mer_fusion_adam (fusion.cu).  MLP is one chain over the concatenation A | T | V; Attention is
// three chains (audio, text, video), a chain over the concat of their outputs, fc_att (no softmax) and the weighted
// sum; both end in the same two heads.  Dropout mask t of the reference's forward order (chain-major, layer-minor)
// acts on that layer's [B, width] output.  fp32 SIMT with a fixed summation order (no atomics on data): results are
// bit-reproducible, eager == CUDA-graph replay.
#include <cooperative_groups.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace cg = cooperative_groups;

namespace {

using namespace mer;

constexpr int CL = 8;       // CTAs per cluster
constexpr int NT = 256;     // threads per CTA
constexpr int NW = NT / 32;
constexpr int RB = 4;       // batch rows per cluster
constexpr int XCH = 3072;   // staging chunk of an input row (floats); also holds the head's d(concat), 3 * 1024 wide
constexpr int MAXC = 4;     // output columns per warp and pass
constexpr int MAXD = MER_MLP_MAX_LAYERS;
constexpr int MAXCH = 4;    // chains: MLP 1, Attention 3 + the attention chain
constexpr int KT = 32;      // input columns per backward tile

struct MlpArgs {
  int kind, D, nch, B, train;
  int K0[MAXCH];            // input width of each chain's first layer
  int N[MAXD];              // layer widths (the same in every chain)
  int L, O1, O2, WM;        // last width, heads, ping-pong buffer row pitch
  int in_dims[3];
  long long w[MAXCH][MAXD], b[MAXCH][MAXD];
  long long att_w, att_b, o1_w, o1_b, o2_w, o2_b;
  const float* P;
  const float* x[3];
  const float* ext_mask[MAXCH * MAXD];
  const long long* emo; const float* val;
  float p_drop, mscale, inv_batch;
  unsigned long long seed;
  const int* step;
  float *features, *emos_out, *vals_out;
  // workspace ([B, .] row-major)
  float* xcat;                          // MLP: the concatenated input A | T | V
  float* hcat;                          // Attention: the concat of the three chains' outputs
  float* act[MAXCH][MAXD];              // each layer's output (after dropout)
  float* g[MAXCH][MAXD];                // gradient w.r.t. each layer's pre-activation
  float *d_att, *d_emos, *d_vals, *loss_terms;
};

struct Plan {  // shared-memory offsets (floats)
  int xs, bA, bB, hcat, red, total;
};

Plan make_plan(const MlpArgs& a) {
  Plan p;
  int o = 0;
  auto take = [&](int n) { int r = o; o += (n + 3) & ~3; return r; };
  p.xs = take(RB * XCH);
  p.bA = take(RB * a.WM);
  p.bB = take(RB * a.WM);
  p.hcat = take(a.kind == 1 ? RB * 3 * a.L : 0);
  p.red = take(NT * RB);
  p.total = o;
  return p;
}

// acc[c][r] += sum_k in[r][k] * W[n_c][k], k in [0, K), for this warp's columns n_c = nb + warp + NW c < n1
__device__ __forceinline__ void mlp_accumulate(float (&acc)[MAXC][RB], const float* __restrict__ in, int ldin, int K,
                                               const float* __restrict__ W, long long ldw, int nb, int n1) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = lane; k < K; k += 32) {
    float xv[RB];
#pragma unroll
    for (int r = 0; r < RB; ++r) xv[r] = in[r * ldin + k];
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      const int n = nb + warp + NW * c;
      if (n < n1) {
        const float w = __ldg(W + (long long)n * ldw + k);
#pragma unroll
        for (int r = 0; r < RB; ++r) acc[c][r] = fmaf(xv[r], w, acc[c][r]);
      }
    }
  }
}

__device__ __forceinline__ float mlp_warp_allsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one input element of chain c's first layer (row < B): the caller's feature, or for the MLP the concat A | T | V
__device__ __forceinline__ float chain_input(const MlpArgs& a, int c, int row, int k) {
  if (a.kind == 1) return a.x[c][(long long)row * a.K0[c] + k];
  if (k < a.in_dims[0]) return a.x[0][(long long)row * a.in_dims[0] + k];
  k -= a.in_dims[0];
  if (k < a.in_dims[1]) return a.x[1][(long long)row * a.in_dims[1] + k];
  k -= a.in_dims[1];
  return a.x[2][(long long)row * a.in_dims[2] + k];
}

// dx[r][k] = sum_n gin[r][n] W[n][k] for this CTA's input columns k in [k0, k1): tiles of KT columns, thread = (k, n-lane),
// the NW n-lane partials summed in lane order; fin(r, k, value) per element (r < RB).
template <class Fin>
__device__ __forceinline__ void mlp_backward_cols(const float* __restrict__ gin, int ldg, int N,
                                                  const float* __restrict__ W, long long ldw, int k0, int k1, float* red,
                                                  Fin fin) {
  const int tid = threadIdx.x, kk = tid % KT, nl = tid / KT;
  constexpr int NL = NT / KT;
  for (int kb = k0; kb < k1; kb += KT) {
    const int k = kb + kk;
    if (k < k1) {
      float acc[RB];
#pragma unroll
      for (int r = 0; r < RB; ++r) acc[r] = 0.f;
#pragma unroll 4
      for (int n = nl; n < N; n += NL) {
        const float w = __ldg(W + (long long)n * ldw + k);
#pragma unroll
        for (int r = 0; r < RB; ++r) acc[r] = fmaf(gin[r * ldg + n], w, acc[r]);
      }
#pragma unroll
      for (int r = 0; r < RB; ++r) red[(nl * RB + r) * KT + kk] = acc[r];
    }
    __syncthreads();
    if (tid < RB * KT) {
      const int r = tid / KT, k2 = kb + tid % KT;
      if (k2 < k1) {
        float s = 0.f;
#pragma unroll
        for (int l = 0; l < NL; ++l) s += red[(l * RB + r) * KT + tid % KT];
        fin(r, k2, s);
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(NT, 1) mlp_rows_kernel(const __grid_constant__ MlpArgs a, const __grid_constant__ Plan pl) {
  extern __shared__ __align__(16) float smem[];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int B = a.B, D = a.D, L = a.L, L3 = 3 * a.L;
  const int row0 = (int)(blockIdx.x / CL) * RB;
  const bool train = a.train != 0;
  const bool drop = train && a.p_drop > 0.f;
  const int step = drop ? *a.step : 0;
  const float* P = a.P;
  float* xs = smem + pl.xs;
  auto bufp = [&](int i) { return i ? smem + pl.bB : smem + pl.bA; };  // the two ping-pong buffers
  float* hcat = smem + pl.hcat;
  float* red = smem + pl.red;
  float* dh = xs;  // Attention: the head's share of d(concat), [RB][3L]; the staged inputs are dead by then

  cluster.sync();  // every CTA of the cluster is running: DSMEM stores may begin
  float* peer_lane = nullptr;  // lanes 0..7 each keep one peer's view of the current output buffer
  int cur = 0;                 // bufp(cur) holds the current layer input

  // ================= forward =================
  for (int c = 0; c < a.nch; ++c) {
    for (int l = 0; l < D; ++l) {
      const int N = a.N[l], K = l == 0 ? a.K0[c] : a.N[l - 1];
      const int HC = (N + CL - 1) / CL;
      const int n0 = min(N, rank * HC), n1 = min(N, n0 + HC);
      const float* W = P + a.w[c][l];
      const float* bias = P + a.b[c][l];
      // where this layer's output goes: the next ping-pong buffer, or (last layer of an Attention modality chain) the
      // concat buffer at column offset c * L
      const bool to_cat = a.kind == 1 && c < 3 && l == D - 1;
      float* out = to_cat ? hcat + c * L : bufp(cur ^ 1);
      const int ldo = to_cat ? L3 : N;
      peer_lane = cluster.map_shared_rank(out, lane & (CL - 1));
      const int mask_id = c * D + l;
      const float* emask = a.ext_mask[mask_id];
      float* gact = a.act[c][l];
      const bool from_global = l == 0 && !(a.kind == 1 && c == 3);
      const float* in = from_global ? xs : (l == 0 ? hcat : bufp(cur));
      const int ldin = from_global ? XCH : (l == 0 ? L3 : K);
      const bool staged_once = from_global && K <= XCH;
      if (staged_once) {
        for (int i = tid; i < RB * K; i += NT) {
          const int r = i / K, k = i % K, row = row0 + r;
          const float v = row < B ? chain_input(a, c, row, k) : 0.f;
          xs[r * XCH + k] = v;
          if (train && a.kind == 0 && rank == 0 && row < B) a.xcat[(long long)row * K + k] = v;
        }
        __syncthreads();
      }
      for (int nb = n0; nb < n1; nb += NW * MAXC) {
        float acc[MAXC][RB];
#pragma unroll
        for (int q = 0; q < MAXC; ++q)
#pragma unroll
          for (int r = 0; r < RB; ++r) acc[q][r] = 0.f;
        if (from_global && !staged_once) {
          for (int kc0 = 0; kc0 < K; kc0 += XCH) {
            const int kc = min(XCH, K - kc0);
            for (int i = tid; i < RB * kc; i += NT) {
              const int r = i / kc, k = i % kc, row = row0 + r;
              const float v = row < B ? chain_input(a, c, row, kc0 + k) : 0.f;
              xs[r * XCH + k] = v;
              if (train && a.kind == 0 && rank == 0 && nb == n0 && row < B) a.xcat[(long long)row * K + kc0 + k] = v;
            }
            __syncthreads();
            mlp_accumulate(acc, xs, XCH, kc, W + kc0, K, nb, n1);
            __syncthreads();
          }
        } else {
          mlp_accumulate(acc, in, ldin, K, W, K, nb, n1);
        }
#pragma unroll
        for (int q = 0; q < MAXC; ++q) {
          const int n = nb + warp + NW * q;
          if (n >= n1) continue;
#pragma unroll
          for (int r = 0; r < RB; ++r) {
            const int row = row0 + r;
            float v = fmaxf(mlp_warp_allsum(acc[q][r]) + bias[n], 0.f);
            if (drop && row < B) {
              const long long i = (long long)row * N + n;
              v *= (emask ? emask[i] : keep_hash(a.seed, mask_id, step, i, a.p_drop)) * a.mscale;
            }
            if (lane < CL) peer_lane[r * ldo + n] = v;
            if (lane == CL + r && train && row < B) {
              gact[(long long)row * N + n] = v;
              if (to_cat) a.hcat[(long long)row * L3 + c * L + n] = v;
            }
          }
        }
      }
      cluster.sync();
      if (!to_cat) cur ^= 1;
    }
  }

  // ================= head (replicated in every CTA, warp r <-> row r) =================
  // MLP: features = bufp(cur) (the chain's output).  Attention: z = bufp(cur) (attention chain output), fused features
  // into bufp(cur ^ 1) rows [0, RB), d features into bufp(cur ^ 1) + RB L.
  float* zb = bufp(cur);
  float* fb = a.kind == 1 ? bufp(cur ^ 1) : bufp(cur);
  float* dfb = a.kind == 1 ? bufp(cur ^ 1) + RB * L : bufp(cur ^ 1);
  const float* w_o1 = P + a.o1_w; const float* b_o1 = P + a.o1_b;
  const float* w_o2 = P + a.o2_w; const float* b_o2 = P + a.o2_b;
  const float* w_att = P + a.att_w; const float* b_att = P + a.att_b;
  const int O1 = a.O1, O2 = a.O2;
  if (warp < RB) {
    const int r = warp, row = row0 + r;
    const bool live = row < B;
    float att[3] = {0.f, 0.f, 0.f};
    if (a.kind == 1) {
      for (int j = lane; j < L; j += 32) {
        const float z = zb[r * L + j];
#pragma unroll
        for (int m = 0; m < 3; ++m) att[m] = fmaf(w_att[m * L + j], z, att[m]);
      }
#pragma unroll
      for (int m = 0; m < 3; ++m) att[m] = mlp_warp_allsum(att[m]) + b_att[m];
      for (int j = lane; j < L; j += 32) {
        const float* h = hcat + r * L3;
        fb[r * L + j] = (h[j] * att[0] + h[L + j] * att[1]) + h[2 * L + j] * att[2];
      }
      __syncwarp();
    }
    float logit[MER_MLP_MAX_OUT1], vout[MER_MLP_MAX_OUT2];
#pragma unroll
    for (int q = 0; q < MER_MLP_MAX_OUT1; ++q) logit[q] = 0.f;
#pragma unroll
    for (int q = 0; q < MER_MLP_MAX_OUT2; ++q) vout[q] = 0.f;
    for (int j = lane; j < L; j += 32) {
      const float f = fb[r * L + j];
      if (rank == 0 && live) a.features[(long long)row * L + j] = f;
#pragma unroll
      for (int q = 0; q < MER_MLP_MAX_OUT1; ++q)
        if (q < O1) logit[q] = fmaf(w_o1[q * L + j], f, logit[q]);
#pragma unroll
      for (int q = 0; q < MER_MLP_MAX_OUT2; ++q)
        if (q < O2) vout[q] = fmaf(w_o2[q * L + j], f, vout[q]);
    }
#pragma unroll
    for (int q = 0; q < MER_MLP_MAX_OUT1; ++q)
      if (q < O1) logit[q] = mlp_warp_allsum(logit[q]) + b_o1[q];
#pragma unroll
    for (int q = 0; q < MER_MLP_MAX_OUT2; ++q)
      if (q < O2) vout[q] = mlp_warp_allsum(vout[q]) + b_o2[q];
    if (rank == 0 && live && lane == 0) {
#pragma unroll
      for (int q = 0; q < MER_MLP_MAX_OUT1; ++q)
        if (q < O1) a.emos_out[(long long)row * O1 + q] = logit[q];
#pragma unroll
      for (int q = 0; q < MER_MLP_MAX_OUT2; ++q)
        if (q < O2) a.vals_out[(long long)row * O2 + q] = vout[q];
    }
    if (train) {
      // CELoss: NLL(log_softmax) summed / N; MSELoss: squared error summed / N (main-release.py:293-315)
      const int tgt = live ? (int)a.emo[row] : 0;
      float mx = logit[0];
#pragma unroll
      for (int q = 1; q < MER_MLP_MAX_OUT1; ++q)
        if (q < O1) mx = fmaxf(mx, logit[q]);
      float se = 0.f;
#pragma unroll
      for (int q = 0; q < MER_MLP_MAX_OUT1; ++q)
        if (q < O1) se += expf(logit[q] - mx);
      const float lse = mx + logf(se);
      float ce = 0.f, mse = 0.f, dlog[MER_MLP_MAX_OUT1], dval[MER_MLP_MAX_OUT2];
#pragma unroll
      for (int q = 0; q < MER_MLP_MAX_OUT1; ++q) {
        dlog[q] = 0.f;
        if (q < O1) {
          if (q == tgt) ce = lse - logit[q];
          dlog[q] = live ? (expf(logit[q] - lse) - (q == tgt ? 1.f : 0.f)) * a.inv_batch : 0.f;
        }
      }
#pragma unroll
      for (int q = 0; q < MER_MLP_MAX_OUT2; ++q) {
        dval[q] = 0.f;
        if (q < O2) {
          const float dd = live ? vout[q] - a.val[(long long)row * O2 + q] : 0.f;
          mse += dd * dd;
          dval[q] = 2.f * dd * a.inv_batch;
        }
      }
      if (rank == 0 && live && lane == 0) {
        a.loss_terms[2 * row] = ce;
        a.loss_terms[2 * row + 1] = mse;
#pragma unroll
        for (int q = 0; q < MER_MLP_MAX_OUT1; ++q)
          if (q < O1) a.d_emos[(long long)row * O1 + q] = dlog[q];
#pragma unroll
        for (int q = 0; q < MER_MLP_MAX_OUT2; ++q)
          if (q < O2) a.d_vals[(long long)row * O2 + q] = dval[q];
      }
      float datt[3] = {0.f, 0.f, 0.f};
      for (int j = lane; j < L; j += 32) {
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < MER_MLP_MAX_OUT1; ++q)
          if (q < O1) s = fmaf(w_o1[q * L + j], dlog[q], s);
#pragma unroll
        for (int q = 0; q < MER_MLP_MAX_OUT2; ++q)
          if (q < O2) s = fmaf(w_o2[q * L + j], dval[q], s);
        if (a.kind == 0) {
          // d features = d (last layer output): through the dropout and the ReLU of the chain's last layer
          const float g = fb[r * L + j] > 0.f ? s * a.mscale : 0.f;
          dfb[r * L + j] = g;
          if (rank == 0 && live) a.g[0][D - 1][(long long)row * L + j] = g;
        } else {
          dfb[r * L + j] = s;
          const float* h = hcat + r * L3;
#pragma unroll
          for (int m = 0; m < 3; ++m) {
            datt[m] = fmaf(h[m * L + j], s, datt[m]);
            dh[r * L3 + m * L + j] = att[m] * s;
          }
        }
      }
      if (a.kind == 1) {
#pragma unroll
        for (int m = 0; m < 3; ++m) datt[m] = mlp_warp_allsum(datt[m]);
        if (rank == 0 && live && lane == 0)
#pragma unroll
          for (int m = 0; m < 3; ++m) a.d_att[3 * row + m] = datt[m];
        for (int j = lane; j < L; j += 32) {
          const float dz = (w_att[j] * datt[0] + w_att[L + j] * datt[1]) + w_att[2 * L + j] * datt[2];
          const float g = zb[r * L + j] > 0.f ? dz * a.mscale : 0.f;
          zb[r * L + j] = g;  // z is dead once its own element has been read
          if (rank == 0 && live) a.g[3][D - 1][(long long)row * L + j] = g;
        }
      }
    }
  }
  // no CTA may exit (eval), or store into a peer's buffers (train), while that peer's head still reads them
  cluster.sync();
  if (!train) return;

  // ================= backward: data gradients =================
  // gcur: the full [RB][N_l] gradient of the current layer's pre-activation (every CTA holds a copy); the layer below's
  // is computed for this CTA's input columns, scaled through its dropout and ReLU, and stored into every peer's copy.
  auto chain_back = [&](int c, const float* gcur, int ldg, int gbuf) {
    for (int l = D - 1; l >= 1; --l) {
      const int N = a.N[l], K = a.N[l - 1];
      const int KC = (K + CL - 1) / CL;
      const int k0 = min(K, rank * KC), k1 = min(K, k0 + KC);
      float* out = bufp(gbuf);
      const float* act = a.act[c][l - 1];
      float* gg = a.g[c][l - 1];
      mlp_backward_cols(gcur, ldg, N, P + a.w[c][l], K, k0, k1, red, [&](int r, int k, float s) {
        const int row = row0 + r;
        const float o = row < B ? act[(long long)row * K + k] : 0.f;
        const float g = o > 0.f ? s * a.mscale : 0.f;
        for (int p = 0; p < CL; ++p) cluster.map_shared_rank(out, p)[r * K + k] = g;
        if (row < B) gg[(long long)row * K + k] = g;
      });
      cluster.sync();
      gcur = out;
      ldg = K;
      gbuf ^= 1;
    }
  };
  if (a.kind == 0) {
    chain_back(0, dfb, L, cur);
  } else {
    // the attention chain, then d(concat) = its first layer's input gradient (through the chain outputs' dropout and
    // ReLU) plus the head's share, written over the concat buffer, then the three modality chains
    chain_back(3, zb, L, cur ^ 1);
    const int g3 = D % 2 == 1 ? cur : cur ^ 1;  // where chain_back left the first layer's gradient
    const float* g0 = bufp(g3);
    const int KC = (L3 + CL - 1) / CL;
    const int k0 = min(L3, rank * KC), k1 = min(L3, k0 + KC);
    mlp_backward_cols(g0, a.N[0], a.N[0], P + a.w[3][0], L3, k0, k1, red, [&](int r, int k, float s) {
      const int row = row0 + r;
      const float h = hcat[r * L3 + k];
      const float g = h > 0.f ? (dh[r * L3 + k] + s) * a.mscale : 0.f;
      for (int p = 0; p < CL; ++p) cluster.map_shared_rank(hcat, p)[r * L3 + k] = g;
      if (row < B) a.g[k / L][D - 1][(long long)row * L + k % L] = g;
    });
    cluster.sync();
    for (int c = 0; c < 3; ++c) {
      chain_back(c, hcat + c * L, L3, 0);
    }
  }
  cluster.sync();
}

struct WProb {
  const float* dy; int lddy;
  const float* x; int ldx;
  int N, K;
  long long w_off, b_off;
  int blk0;
};
constexpr int MAXP = MAXCH * MAXD + 3;

struct WArgs {
  WProb p[MAXP];
  int np, B;
  float* G;
  const float* loss_terms; float inv_batch; float* loss_out;
};

// dW[n, k] = sum_b dy[b, n] x[b, k] and db[n] = sum_b dy[b, n], b in order
__global__ void __launch_bounds__(NT) mlp_wgrad_kernel(const __grid_constant__ WArgs a) {
  const int tid = threadIdx.x;
  int pi = 0;
  for (int i = 1; i < a.np; ++i)
    if ((int)blockIdx.x >= a.p[i].blk0) pi = i;
  const WProb& p = a.p[pi];
  const long long e = (long long)(blockIdx.x - p.blk0) * NT + tid;
  if (e < (long long)p.N * p.K) {
    const int n = (int)(e / p.K), k = (int)(e % p.K);
    float acc = 0.f, accb = 0.f;
#pragma unroll 8
    for (int b = 0; b < a.B; ++b) {
      const float g = p.dy[(long long)b * p.lddy + n];
      accb += g;
      acc = fmaf(g, p.x[(long long)b * p.ldx + k], acc);
    }
    a.G[p.w_off + e] = acc;
    if (k == 0) a.G[p.b_off + n] = accb;
  }
  if (blockIdx.x == 0 && tid == 0) {
    float ce = 0.f, mse = 0.f;
    for (int b = 0; b < a.B; ++b) { ce += a.loss_terms[2 * b]; mse += a.loss_terms[2 * b + 1]; }
    a.loss_out[0] = ce * a.inv_batch;
    a.loss_out[1] = mse * a.inv_batch;
    a.loss_out[2] = ce * a.inv_batch + mse * a.inv_batch;
  }
}

struct Layout {
  long long w[MAXCH][MAXD], b[MAXCH][MAXD];
  long long att_w, att_b, o1_w, o1_b, o2_w, o2_b, total;
  int nch, K0[MAXCH];
};

int check_dims(const MerMlpDims* d) {
  MER_REQUIRE(d, "mer_mlp: null dims");
  MER_REQUIRE(d->kind == MER_MLP_KIND_MLP || d->kind == MER_MLP_KIND_ATTENTION,
              "mer_mlp: kind %d is neither MER_MLP_KIND_MLP (0) nor MER_MLP_KIND_ATTENTION (1)", d->kind);
  MER_REQUIRE(d->n_layers >= 1 && d->n_layers <= MAXD, "mer_mlp: %d layers (1..%d)", d->n_layers, MAXD);
  for (int l = 0; l < d->n_layers; ++l)
    MER_REQUIRE(d->layers[l] >= 1 && d->layers[l] <= MER_MLP_MAX_WIDTH, "mer_mlp: layer %d has width %d (1..%d)", l,
                d->layers[l], MER_MLP_MAX_WIDTH);
  const int in[3] = {d->audio_dim, d->text_dim, d->video_dim};
  for (int m = 0; m < 3; ++m)
    MER_REQUIRE(in[m] >= 1 && in[m] <= MER_MLP_MAX_INPUT, "mer_mlp: input width %d of modality %d (1..%d)", in[m], m,
                MER_MLP_MAX_INPUT);
  MER_REQUIRE(d->out1 >= 1 && d->out1 <= MER_MLP_MAX_OUT1, "mer_mlp: out1 %d (1..%d emotion classes)", d->out1,
              MER_MLP_MAX_OUT1);
  MER_REQUIRE(d->out2 >= 1 && d->out2 <= MER_MLP_MAX_OUT2, "mer_mlp: out2 %d (1..%d valence outputs)", d->out2,
              MER_MLP_MAX_OUT2);
  return 0;
}

int check_batch(const MerMlpDims* d, int B) {
  MER_REQUIRE(B >= 1 && B <= 65535, "mer_mlp: batch %d out of range (1..65535)", B);
  MER_REQUIRE(d->kind != MER_MLP_KIND_ATTENTION || B >= 2,
              "mer_mlp: the Attention net needs at least 2 rows per batch (the reference squeezes a 1-row batch's "
              "fused features to a vector and fails)");
  return 0;
}

Layout make_layout(const MerMlpDims& d) {
  Layout L;
  memset(&L, 0, sizeof(L));
  long long o = 0;
  const int D = d.n_layers, Ll = d.layers[D - 1];
  if (d.kind == MER_MLP_KIND_MLP) {
    L.nch = 1;
    L.K0[0] = d.audio_dim + d.text_dim + d.video_dim;
  } else {
    L.nch = 4;
    L.K0[0] = d.audio_dim; L.K0[1] = d.text_dim; L.K0[2] = d.video_dim; L.K0[3] = 3 * Ll;
  }
  for (int c = 0; c < L.nch; ++c) {
    int K = L.K0[c];
    for (int l = 0; l < D; ++l) {
      L.w[c][l] = o; o += (long long)d.layers[l] * K;
      L.b[c][l] = o; o += d.layers[l];
      K = d.layers[l];
    }
  }
  if (d.kind == MER_MLP_KIND_ATTENTION) {
    L.att_w = o; o += 3ll * Ll;
    L.att_b = o; o += 3;
  }
  L.o1_w = o; o += (long long)d.out1 * Ll;
  L.o1_b = o; o += d.out1;
  L.o2_w = o; o += (long long)d.out2 * Ll;
  L.o2_b = o; o += d.out2;
  L.total = o;
  return L;
}

long long ws_floats(const MerMlpDims& d, int B) {
  const Layout L = make_layout(d);
  const int Ll = d.layers[d.n_layers - 1];
  long long per_row = 0;
  auto r4 = [](long long n) { return (n + 3) / 4 * 4; };
  per_row += d.kind == MER_MLP_KIND_MLP ? L.K0[0] : 3ll * Ll;
  for (int l = 0; l < d.n_layers; ++l) per_row += 2ll * L.nch * d.layers[l];
  per_row += 3 + d.out1 + d.out2 + 2;
  return r4((long long)B * per_row) + 4 * (2 * MAXCH * MAXD + 8) + 64;
}

int fill(MlpArgs& a, const MerMlpDims* d, const float* params, const float* audios, const float* texts,
         const float* videos, int B, void* workspace, long long workspace_bytes, float* features, float* emos_out,
         float* vals_out) {
  if (int rc = check_dims(d)) return rc;
  if (int rc = check_batch(d, B)) return rc;
  MER_REQUIRE(params && audios && texts && videos && workspace && features && emos_out && vals_out,
              "mer_mlp: null operand");
  MER_REQUIRE(workspace_bytes >= ws_floats(*d, B) * 4, "mer_mlp: workspace of %lld bytes, %lld needed",
              workspace_bytes, ws_floats(*d, B) * 4);
  memset(&a, 0, sizeof(a));
  const Layout L = make_layout(*d);
  a.kind = d->kind;
  a.D = d->n_layers;
  a.nch = L.nch;
  a.B = B;
  a.L = d->layers[d->n_layers - 1];
  a.O1 = d->out1;
  a.O2 = d->out2;
  a.WM = 0;
  for (int l = 0; l < a.D; ++l) {
    a.N[l] = d->layers[l];
    a.WM = a.N[l] > a.WM ? a.N[l] : a.WM;
  }
  if (a.kind == MER_MLP_KIND_ATTENTION && 2 * a.L > a.WM) a.WM = 2 * a.L;  // fused features + their gradient
  for (int c = 0; c < MAXCH; ++c) {
    a.K0[c] = L.K0[c];
    for (int l = 0; l < MAXD; ++l) { a.w[c][l] = L.w[c][l]; a.b[c][l] = L.b[c][l]; }
  }
  a.att_w = L.att_w; a.att_b = L.att_b; a.o1_w = L.o1_w; a.o1_b = L.o1_b; a.o2_w = L.o2_w; a.o2_b = L.o2_b;
  a.in_dims[0] = d->audio_dim; a.in_dims[1] = d->text_dim; a.in_dims[2] = d->video_dim;
  a.P = params;
  a.x[0] = audios; a.x[1] = texts; a.x[2] = videos;
  a.features = features; a.emos_out = emos_out; a.vals_out = vals_out;
  a.mscale = 1.f;
  // workspace carve (16-byte aligned pieces)
  float* p = static_cast<float*>(workspace);
  auto take = [&](long long n) { float* r = p; p += (n + 3) / 4 * 4; return r; };
  a.xcat = d->kind == MER_MLP_KIND_MLP ? take((long long)B * L.K0[0]) : nullptr;
  a.hcat = d->kind == MER_MLP_KIND_ATTENTION ? take(3ll * B * a.L) : nullptr;
  for (int c = 0; c < a.nch; ++c)
    for (int l = 0; l < a.D; ++l) {
      a.act[c][l] = take((long long)B * a.N[l]);
      a.g[c][l] = take((long long)B * a.N[l]);
    }
  a.d_att = take(3ll * B);
  a.d_emos = take((long long)B * a.O1);
  a.d_vals = take((long long)B * a.O2);
  a.loss_terms = take(2ll * B);
  return 0;
}

int launch_rows(const MlpArgs& a, cudaStream_t st) {
  static MerPerDevice once;
  const Plan pl = make_plan(a);
  const size_t smem = (size_t)pl.total * 4;
  MER_REQUIRE(smem <= 227 * 1024, "mer_mlp: shared-memory plan of %zu bytes", smem);
  if (once.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(mlp_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    once.mark();
  }
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
  MER_CUDA_CHECK(cudaLaunchKernelEx(&cfg, mlp_rows_kernel, a, pl));
  mer_count_launches(1);
  return 0;
}

int launch_wgrad(const MlpArgs& a, const Layout& L, float* grads, float* loss_out, cudaStream_t st) {
  WArgs w;
  memset(&w, 0, sizeof(w));
  int blk = 0;
  auto add = [&](const float* dy, int lddy, const float* x, int ldx, int N, int K, long long w_off, long long b_off) {
    w.p[w.np] = WProb{dy, lddy, x, ldx, N, K, w_off, b_off, blk};
    blk += (int)(((long long)N * K + NT - 1) / NT);
    ++w.np;
  };
  for (int c = 0; c < a.nch; ++c)
    for (int l = 0; l < a.D; ++l) {
      const float* x;
      int K;
      if (l > 0) { x = a.act[c][l - 1]; K = a.N[l - 1]; }
      else if (a.kind == MER_MLP_KIND_MLP) { x = a.xcat; K = a.K0[0]; }
      else if (c < 3) { x = a.x[c]; K = a.K0[c]; }
      else { x = a.hcat; K = 3 * a.L; }
      add(a.g[c][l], a.N[l], x, K, a.N[l], K, L.w[c][l], L.b[c][l]);
    }
  if (a.kind == MER_MLP_KIND_ATTENTION) add(a.d_att, 3, a.act[3][a.D - 1], a.L, 3, a.L, L.att_w, L.att_b);
  add(a.d_emos, a.O1, a.features, a.L, a.O1, a.L, L.o1_w, L.o1_b);
  add(a.d_vals, a.O2, a.features, a.L, a.O2, a.L, L.o2_w, L.o2_b);
  w.B = a.B;
  w.G = grads;
  w.loss_terms = a.loss_terms;
  w.inv_batch = a.inv_batch;
  w.loss_out = loss_out;
  mlp_wgrad_kernel<<<blk, NT, 0, st>>>(w);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

}  // namespace

extern "C" {

long long mer_mlp_param_count(const MerMlpDims* d) {
  if (check_dims(d)) return -1;
  return make_layout(*d).total;
}

long long mer_mlp_workspace_bytes(const MerMlpDims* d, int max_batch) {
  if (check_dims(d) || check_batch(d, max_batch)) return -1;
  return ws_floats(*d, max_batch) * 4;
}

int mer_mlp_forward(const MerMlpDims* d, const float* params, const float* audios, const float* texts,
                    const float* videos, int batch, void* workspace, long long workspace_bytes, float* features,
                    float* emos_out, float* vals_out, void* stream) {
  MlpArgs a;
  if (int rc = fill(a, d, params, audios, texts, videos, batch, workspace, workspace_bytes, features, emos_out,
                    vals_out))
    return rc;
  a.train = 0;
  return launch_rows(a, static_cast<cudaStream_t>(stream));
}

int mer_mlp_train_step(const MerMlpDims* d, float* params, float* grads, float* exp_avg, float* exp_avg_sq,
                       const float* audios, const float* texts, const float* videos, const int64_t* emos,
                       const float* vals, int batch, float dropout_p, unsigned long long seed, int* step_counter,
                       const float* const* ext_masks, const MerAdamHyper* adam, void* workspace,
                       long long workspace_bytes, float* loss_out, float* features, float* emos_out, float* vals_out,
                       void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MlpArgs a;
  if (int rc = fill(a, d, params, audios, texts, videos, batch, workspace, workspace_bytes, features, emos_out,
                    vals_out))
    return rc;
  MER_REQUIRE(grads && emos && vals && loss_out && step_counter, "mer_mlp_train_step: null operand");
  MER_REQUIRE(!adam || (exp_avg && exp_avg_sq), "mer_mlp_train_step: Adam needs exp_avg and exp_avg_sq");
  MER_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "mer_mlp_train_step: dropout %f (0 <= p < 1)", dropout_p);
  a.train = 1;
  a.emo = reinterpret_cast<const long long*>(emos);
  a.val = vals;
  a.inv_batch = 1.f / (float)batch;
  a.p_drop = dropout_p;
  a.mscale = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
  a.seed = seed;
  a.step = step_counter;
  if (ext_masks)
    for (int m = 0; m < a.nch * a.D; ++m) a.ext_mask[m] = ext_masks[m];
  if (int rc = launch_rows(a, st)) return rc;
  const Layout L = make_layout(*d);
  if (int rc = launch_wgrad(a, L, grads, loss_out, st)) return rc;
  if (!adam) return 0;
  return mer_fusion_adam(params, grads, exp_avg, exp_avg_sq, L.total, adam->lr, adam->beta1, adam->beta2, adam->eps,
                         adam->weight_decay, 1.f, adam->grad_clip, step_counter, stream);
}

}  // extern "C"
