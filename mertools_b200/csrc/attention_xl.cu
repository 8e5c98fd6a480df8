// attention_xl.cu — XLNet's relative self-attention (HF XLNetRelativeAttention.rel_attn_core, attn_type "bi", the
// content stream only, head_dim 64) for packed variable-length sentences:
//
//   score[i, j] = scale * ( (q_i + r_w_bias) . k_j  +  (q_i + r_r_bias) . R[row(i - j)]
//                           + (q_i + r_s_bias) . seg_embed[type_i != type_j] ),         ctx_i = softmax_j . V
//
// i, j count from the sentence start.  R is the layer's projection of the sinusoidal relative-position rows
// ([rows, heads*64]); row(d) is the caller's map from a distance to a table row (clamp_len), given as
// rel_row[d + max_seqlen - 1].  The segment term is present only when the caller passes token types.  Reads the q | k
// rows and V^T the QKV GEMM writes, in the two operand formats of attention_f16.cu: fp16 (mma m16n8k16) and
// tf32-rounded fp32 (mma m16n8k8).
//
// Layout as attention_rel.cu: one CTA = (64-query block, head, sentence), 4 warps x 16 query rows.  A 64 x 64 (query,
// key) tile sees the 127 distances i0 - j0 - 63 .. i0 - j0 + 63; per key tile the CTA gathers those rows of R into
// shared memory, computes C1 = Q Rwin^T (64 x 128, fp32) next to S = Q K^T, and adds C1[i][w] with
// w = (i - i0) - (j - j0) + 63 to S.  The biases are never added to the operand-format q: their products are separate
// fp32 dot products over the operands, r_w_bias . k_j per key and r_r_bias . Rwin[w] per window row (one warp-reduced
// dot per row and tile), and the two segment scalars (q_i + r_s_bias) . seg_embed[0 | 1] per query once per CTA, so
// the result carries no rounding beyond that of q, k, R and P.  Single-buffered: one cp.async group per key tile.
#include <cuda_fp16.h>
#include <stdint.h>

#include "attention_mma.cuh"
#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int HD = 64;
constexpr int BQ = 64;
constexpr int BKV = 64;
constexpr int WIN = 128;  // window rows per key tile (127 used)
constexpr int LDC = WIN + 4;
constexpr int THREADS = 128;

template <bool F16>
struct XlCfg {
  static constexpr int kElem = F16 ? 2 : 4;
  static constexpr int kPerChunk = 16 / kElem;
  static constexpr int kLds = F16 ? 72 : 68;
  static constexpr int kTile = BKV * kLds;  // K or V^T tile
  static constexpr int kWin = WIN * kLds;   // R window
  // K, V^T, R window; C1; r_w_bias . k per key, r_r_bias . R per window row; key token types
  static constexpr int kSmem = (2 * kTile + kWin) * kElem + BQ * LDC * 4 + (BKV + WIN) * 4 + BKV * 4;
};

// elements 2 lane, 2 lane + 1 of a 64-wide operand row, as fp32
template <bool F16, typename T>
__device__ __forceinline__ float2 pair_f32(const T* row, int lane) {
  if constexpr (F16)
    return __half22float2(*reinterpret_cast<const __half2*>(row + 2 * lane));
  else
    return *reinterpret_cast<const float2*>(row + 2 * lane);
}

__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// out_mode: 0 fp32, 1 tf32-rounded fp32, 2 bf16 hi | lo split rows, 3 fp16
template <bool F16>
__global__ void __launch_bounds__(THREADS, 1)
xlnet_attention_kernel(const void* __restrict__ qkv_, const void* __restrict__ vt_, long long vt_ld,
                       const void* __restrict__ r_, long long r_ld, const int* __restrict__ rel_row,
                       const float* __restrict__ r_w_bias, const float* __restrict__ r_r_bias,
                       const float* __restrict__ r_s_bias, const float* __restrict__ seg_embed,
                       const int* __restrict__ token_type, float scale, void* __restrict__ ctx,
                       const int* __restrict__ cu_seqlens, long long tokens, int max_seqlen, int heads, int out_mode) {
  using Cfg = XlCfg<F16>;
  using T = typename std::conditional<F16, uint16_t, float>::type;
  constexpr int LDS = Cfg::kLds;
  constexpr int KS = F16 ? 4 : 8;
  extern __shared__ __align__(16) uint8_t smem_xl[];
  T* Ks = reinterpret_cast<T*>(smem_xl);  // [BKV][LDS]
  T* Vs = Ks + Cfg::kTile;                // [HD][LDS]: V^T, keys along the row
  T* Rw = Vs + Cfg::kTile;                // [WIN][LDS]
  float* C1 = reinterpret_cast<float*>(Rw + Cfg::kWin);  // [BQ][LDC]: q_i . Rwin[w]
  float* kb = C1 + BQ * LDC;                              // [BKV]: r_w_bias . k_j
  float* rb = kb + BKV;                                   // [WIN]: r_r_bias . Rwin[w]
  int* tk = reinterpret_cast<int*>(rb + WIN);             // [BKV]: token type of key j

  const int seq = blockIdx.z, h = blockIdx.y;
  const int start = cu_seqlens[seq];
  const int len = cu_seqlens[seq + 1] - start;
  const int q0 = blockIdx.x * BQ;
  if (q0 >= len) return;
  const int kstart = start & ~7, shift = start - kstart;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const long long ld = 3ll * heads * HD;
  const T* qkv = static_cast<const T*>(qkv_);
  const T* qbase = qkv + (long long)start * ld + h * HD;
  const T* kbase = qkv + heads * HD + h * HD;  // row = absolute token index
  const T* vtbase = static_cast<const T*>(vt_) + (long long)h * HD * vt_ld;
  const T* rbase = static_cast<const T*>(r_) + h * HD;
  const int max_idx = 2 * max_seqlen - 2;
  const bool segs = token_type != nullptr;

  uint32_t qa[KS][4];
  const int row_lo = q0 + warp * 16 + g, row_hi = row_lo + 8;
  load_a<F16>(qa, qbase + (long long)min(row_lo, len - 1) * ld, qbase + (long long)min(row_hi, len - 1) * ld, t);
  const float2 bw = *reinterpret_cast<const float2*>(r_w_bias + h * HD + 2 * lane);
  const float2 br = *reinterpret_cast<const float2*>(r_r_bias + h * HD + 2 * lane);

  // segment scalars e[s] = (q_i + r_s_bias) . seg_embed[s] of this thread's rows lo / hi, and their token types
  float e0_lo = 0.f, e1_lo = 0.f, e0_hi = 0.f, e1_hi = 0.f;
  int tt_lo = 0, tt_hi = 0;
  if (segs) {
    const float2 bs = *reinterpret_cast<const float2*>(r_s_bias + h * HD + 2 * lane);
    const float2 s0 = *reinterpret_cast<const float2*>(seg_embed + h * HD + 2 * lane);
    const float2 s1 = *reinterpret_cast<const float2*>(seg_embed + (heads + h) * HD + 2 * lane);
    for (int r = 0; r < 16; ++r) {
      const float2 q = pair_f32<F16>(qbase + (long long)min(q0 + warp * 16 + r, len - 1) * ld, lane);
      const float x = q.x + bs.x, y = q.y + bs.y;
      const float p0 = warp_sum(x * s0.x + y * s0.y), p1 = warp_sum(x * s1.x + y * s1.y);
      if (g == r) e0_lo = p0, e1_lo = p1;
      if (g + 8 == r) e0_hi = p0, e1_hi = p1;
    }
    tt_lo = token_type[start + min(row_lo, len - 1)];
    tt_hi = token_type[start + min(row_hi, len - 1)];
  }

  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  const int n_kv = (shift + len + BKV - 1) / BKV;
  const float SL2 = scale * 1.4426950408889634f;
  constexpr int CPR = HD / Cfg::kPerChunk;  // 16-byte chunks per 64-element row

  for (int j = 0; j < n_kv; ++j) {
    const int p0 = kstart + j * BKV;  // absolute token index of tile column 0
    const int rel0 = j * BKV - shift; // its index inside the sentence
    // window row w holds distance d = q0 - rel0 - 63 + w
    const int d0 = q0 - rel0 - (BKV - 1);
#pragma unroll
    for (int i = 0; i < BKV * CPR / THREADS; ++i) {
      const int idx = tid + i * THREADS;
      const int r = idx / CPR, c = (idx % CPR) * Cfg::kPerChunk;
      const int key = p0 + r;
      const bool kin = key >= start && key < start + len;
      cp_async16(Ks + r * LDS + c, kbase + (long long)(kin ? key : start) * ld + c, kin ? 16 : 0);
      const long long vk = p0 + c;
      const int vbytes = vk >= tokens ? 0 : (int)min(16ll, (tokens - vk) * Cfg::kElem);
      cp_async16(Vs + r * LDS + c, vtbase + (long long)r * vt_ld + (vbytes ? vk : 0), vbytes);
    }
#pragma unroll
    for (int i = 0; i < WIN * CPR / THREADS; ++i) {
      const int idx = tid + i * THREADS;
      const int w = idx / CPR, c = (idx % CPR) * Cfg::kPerChunk;
      const long long row = __ldg(rel_row + min(max(d0 + w + max_seqlen - 1, 0), max_idx));
      cp_async16(Rw + w * LDS + c, rbase + row * r_ld + c, 16);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    if (segs && tid < BKV) {
      const int key = p0 + tid;
      tk[tid] = (key >= start && key < start + len) ? __ldg(token_type + key) : 0;
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();

    // ---- S = Q K^T (16 x 64 per warp) ----
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) mma_row8<F16, T, LDS>(s[nt], qa, Ks + nt * 8 * LDS, g, t);
    // ---- C1 = Q Rwin^T (this warp's 16 rows) ----
    {
      const int r = warp * 16 + g;
#pragma unroll 4
      for (int nt = 0; nt < WIN / 8; ++nt) {
        float c[4];
        mma_row8<F16, T, LDS>(c, qa, Rw + nt * 8 * LDS, g, t);
        *reinterpret_cast<float2*>(C1 + r * LDC + nt * 8 + 2 * t) = make_float2(c[0], c[1]);
        *reinterpret_cast<float2*>(C1 + (r + 8) * LDC + nt * 8 + 2 * t) = make_float2(c[2], c[3]);
      }
    }
    // ---- bias products in fp32: kb[j] = r_w_bias . k_j (16 keys per warp), rb[w] = r_r_bias . Rwin[w] (32 rows) ----
    for (int r = 0; r < 16; ++r) {
      const int jj = warp * 16 + r;
      const float2 k = pair_f32<F16>(Ks + jj * LDS, lane);
      const float p = warp_sum(k.x * bw.x + k.y * bw.y);
      if (lane == 0) kb[jj] = p;
    }
    for (int r = 0; r < WIN / 4; ++r) {
      const int w = warp * (WIN / 4) + r;
      const float2 x = pair_f32<F16>(Rw + w * LDS, lane);
      const float p = warp_sum(x.x * br.x + x.y * br.y);
      if (lane == 0) rb[w] = p;
    }
    __syncthreads();
    // ---- S += kb[j] + C1[i][w] + rb[w] (+ segment term), w = i - j + 63; mask keys outside the sentence ----
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = warp * 16 + g + (e >> 1) * 8, jj = nt * 8 + 2 * t + (e & 1);
        const int w = i - jj + (BKV - 1);
        const int k = rel0 + jj;
        float x = s[nt][e] + kb[jj] + C1[i * LDC + w] + rb[w];
        if (segs) {
          const bool hi = e >> 1;
          const bool diff = (hi ? tt_hi : tt_lo) != tk[jj];
          x += diff ? (hi ? e1_hi : e1_lo) : (hi ? e0_hi : e0_lo);
        }
        s[nt][e] = (k < 0 || k >= len) ? -INFINITY : x;
      }
    }
    // ---- online softmax (base 2, scale folded in) ----
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx_lo = fmaxf(mx_lo, fmaxf(s[nt][0], s[nt][1]));
      mx_hi = fmaxf(mx_hi, fmaxf(s[nt][2], s[nt][3]));
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
    const float mn_lo = fmaxf(m_lo, mx_lo), mn_hi = fmaxf(m_hi, mx_hi);
    // every row has a valid key in its first tile, so mn is finite from there on
    const float sc_lo = fast_ex2((m_lo - mn_lo) * SL2), sc_hi = fast_ex2((m_hi - mn_hi) * SL2);
    m_lo = mn_lo;
    m_hi = mn_hi;
    const float b_lo = mn_lo * SL2, b_hi = mn_hi * SL2;
    float ps_lo = 0.f, ps_hi = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = fast_ex2(fmaf(s[nt][0], SL2, -b_lo));
      s[nt][1] = fast_ex2(fmaf(s[nt][1], SL2, -b_lo));
      s[nt][2] = fast_ex2(fmaf(s[nt][2], SL2, -b_hi));
      s[nt][3] = fast_ex2(fmaf(s[nt][3], SL2, -b_hi));
      ps_lo += s[nt][0] + s[nt][1];
      ps_hi += s[nt][2] + s[nt][3];
    }
    l_lo = l_lo * sc_lo + ps_lo;
    l_hi = l_hi * sc_hi + ps_hi;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      o[dt][0] *= sc_lo; o[dt][1] *= sc_lo; o[dt][2] *= sc_hi; o[dt][3] *= sc_hi;
    }
    // ---- O += P V ----
    if (F16) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {  // 16 keys per step: n-tiles 2 ks and 2 ks + 1 of S
        uint32_t pa[4];
        pa[0] = pack_f16x2(s[2 * ks][0], s[2 * ks][1]);
        pa[1] = pack_f16x2(s[2 * ks][2], s[2 * ks][3]);
        pa[2] = pack_f16x2(s[2 * ks + 1][0], s[2 * ks + 1][1]);
        pa[3] = pack_f16x2(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
        for (int dt = 0; dt < 8; ++dt) {
          const uint32_t* w = reinterpret_cast<const uint32_t*>(Vs + (dt * 8 + g) * LDS + ks * 16);
          mma_f16(o[dt], pa, w[t], w[t + 4]);
        }
      }
    } else {
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {  // keys 2t / 2t+1 of the group <-> k-columns t / t+4
        uint32_t pa[4];
        pa[0] = __float_as_uint(round_tf32(s[ks][0]));
        pa[1] = __float_as_uint(round_tf32(s[ks][2]));
        pa[2] = __float_as_uint(round_tf32(s[ks][1]));
        pa[3] = __float_as_uint(round_tf32(s[ks][3]));
#pragma unroll
        for (int dt = 0; dt < 8; ++dt) {
          const float2 w = *reinterpret_cast<const float2*>(
              reinterpret_cast<const float*>(Vs) + (dt * 8 + g) * LDS + ks * 8 + 2 * t);
          mma_tf32(o[dt], pa, __float_as_uint(w.x), __float_as_uint(w.y));
        }
      }
    }
    __syncthreads();  // everyone is done with the tiles, C1, kb, rb and tk before the next key tile overwrites them
  }

  // ---- finalize ----
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
  const float inv_lo = 1.0f / l_lo, inv_hi = 1.0f / l_hi;
  const long long ldc = (long long)heads * HD;
#pragma unroll
  for (int dt = 0; dt < 8; ++dt) {
    const int col = h * HD + dt * 8 + 2 * t;
    float2 a = make_float2(o[dt][0] * inv_lo, o[dt][1] * inv_lo);
    float2 b = make_float2(o[dt][2] * inv_hi, o[dt][3] * inv_hi);
    const long long r_lo = (long long)(start + row_lo) * ldc, r_hi = (long long)(start + row_hi) * ldc;
    if (out_mode == 3) {
      uint16_t* c16 = static_cast<uint16_t*>(ctx);
      if (row_lo < len) *reinterpret_cast<uint32_t*>(c16 + r_lo + col) = pack_f16x2(a.x, a.y);
      if (row_hi < len) *reinterpret_cast<uint32_t*>(c16 + r_hi + col) = pack_f16x2(b.x, b.y);
      continue;
    }
    float* c32 = static_cast<float*>(ctx);
    if (out_mode == 2) {  // split bf16 rows for a BF16X3 out-proj GEMM
      if (row_lo < len) store_split2(c32 + r_lo, col, a.x, a.y);
      if (row_hi < len) store_split2(c32 + r_hi, col, b.x, b.y);
      continue;
    }
    if (out_mode == 1) {
      a.x = round_tf32(a.x); a.y = round_tf32(a.y); b.x = round_tf32(b.x); b.y = round_tf32(b.y);
    }
    if (row_lo < len) *reinterpret_cast<float2*>(c32 + r_lo + col) = a;
    if (row_hi < len) *reinterpret_cast<float2*>(c32 + r_hi + col) = b;
  }
}

template <bool F16>
int launch_xl(const void* qkv, const void* vt, long long vt_ld, const void* r, long long r_ld, const int32_t* rel_row,
              const float* r_w_bias, const float* r_r_bias, const float* r_s_bias, const float* seg_embed,
              const int32_t* token_type, float scale, void* ctx, const int32_t* cu_seqlens, int n_seq,
              long long tokens, int max_seqlen, int heads, int out_mode, cudaStream_t stream) {
  using Cfg = XlCfg<F16>;
  static MerPerDevice attr_set;
  if (attr_set.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(xlnet_attention_kernel<F16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        Cfg::kSmem));
    attr_set.mark();
  }
  dim3 grid((max_seqlen + BQ - 1) / BQ, heads, n_seq);
  xlnet_attention_kernel<F16><<<grid, THREADS, Cfg::kSmem, stream>>>(
      qkv, vt, vt_ld, r, r_ld, rel_row, r_w_bias, r_r_bias, r_s_bias, seg_embed, token_type, scale, ctx, cu_seqlens,
      tokens, max_seqlen, heads, out_mode);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

}  // namespace

extern "C" int mer_xlnet_attention(const void* qkv, const void* vt, long long vt_ld, const void* r, long long r_ld,
                                   const int32_t* rel_row, const float* r_w_bias, const float* r_r_bias,
                                   const float* r_s_bias, const float* seg_embed, const int32_t* token_type,
                                   float scale, void* ctx, const int32_t* cu_seqlens, int n_seq, long long tokens,
                                   int max_seqlen, int heads, int flags, void* stream_) {
  const char* name = "mer_xlnet_attention";
  const bool f16 = (flags & MER_ATT_QKV_F16) != 0;
  const int out_flags = flags & ~MER_ATT_QKV_F16;
  MER_REQUIRE(out_flags == 0 || out_flags == MER_EPI_ROUND_TF32 || out_flags == MER_EPI_SPLIT_BF16 ||
                  out_flags == MER_EPI_OUT_F16,
              "%s: flags %d (MER_ATT_QKV_F16 and at most one of MER_EPI_ROUND_TF32 / MER_EPI_SPLIT_BF16 / "
              "MER_EPI_OUT_F16)", name, flags);
  MER_REQUIRE(qkv && vt && ctx && cu_seqlens, "%s: null operand", name);
  MER_REQUIRE(r && rel_row, "%s: null relative-position table (r or rel_row)", name);
  MER_REQUIRE(r_w_bias && r_r_bias && r_s_bias && seg_embed, "%s: null bias (r_w_bias, r_r_bias, r_s_bias or "
              "seg_embed)", name);
  MER_REQUIRE(heads > 0 && heads <= 65535, "%s: heads %d (1 .. 65535)", name, heads);
  MER_REQUIRE(n_seq > 0 && n_seq <= 65535, "%s: n_seq %d (1 .. 65535)", name, n_seq);
  const int per_chunk = f16 ? 8 : 4;
  MER_REQUIRE(vt_ld >= tokens && vt_ld % per_chunk == 0, "%s: V^T pitch %lld must be a multiple of %d >= tokens %lld",
              name, vt_ld, per_chunk, tokens);
  MER_REQUIRE(r_ld >= (long long)heads * HD && r_ld % per_chunk == 0,
              "%s: R pitch %lld must be a multiple of %d >= heads * 64", name, r_ld, per_chunk);
  MER_REQUIRE(aligned16(qkv) && aligned16(vt) && aligned16(r), "%s: qkv, vt and r must be 16-byte aligned", name);
  MER_REQUIRE(aligned8(r_w_bias) && aligned8(r_r_bias) && aligned8(r_s_bias) && aligned8(seg_embed),
              "%s: r_w_bias, r_r_bias, r_s_bias and seg_embed must be 8-byte aligned", name);
  MER_REQUIRE(max_seqlen > 0 && max_seqlen <= tokens, "%s: max_seqlen %d (1 .. tokens %lld)", name, max_seqlen,
              tokens);
  const int out_mode = out_flags == MER_EPI_OUT_F16 ? 3 : out_flags == MER_EPI_SPLIT_BF16 ? 2
                       : out_flags == MER_EPI_ROUND_TF32 ? 1 : 0;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (f16)
    return launch_xl<true>(qkv, vt, vt_ld, r, r_ld, rel_row, r_w_bias, r_r_bias, r_s_bias, seg_embed, token_type,
                           scale, ctx, cu_seqlens, n_seq, tokens, max_seqlen, heads, out_mode, stream);
  return launch_xl<false>(qkv, vt, vt_ld, r, r_ld, rel_row, r_w_bias, r_r_bias, r_s_bias, seg_embed, token_type,
                          scale, ctx, cu_seqlens, n_seq, tokens, max_seqlen, heads, out_mode, stream);
}
