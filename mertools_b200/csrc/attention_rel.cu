// attention_rel.cu — DeBERTa's disentangled self-attention (HF DisentangledSelfAttention, deberta and deberta-v2,
// pos_att_type c2p | p2c, head_dim 64) for packed variable-length sentences:
//
//   score[i, j] = scale * ( q_i . k_j  +  q_i . PK[row(i - j)]  +  k_j . PQ[row(i - j)] ),   ctx_i = softmax_j . V
//
// i, j count from the sentence start.  PK / PQ are the layer's projections of the relative-position table
// ([2 span, heads*64] each); row(d) is the caller's map from a relative distance to a table row (v1: clamped
// distance, v2: clamped log bucket), given as rel_row[d + max_seqlen - 1].  Reads the q | k rows and V^T the QKV GEMM
// writes, in the two operand formats of attention_f16.cu: fp16 (mma m16n8k16) and tf32-rounded fp32 (mma m16n8k8).
//
// One CTA = (64-query block, head, sentence), 4 warps x 16 query rows, as attention_vt_kernel.  A 64 x 64 (query, key)
// tile only sees the 127 relative distances i0 - j0 - 63 .. i0 - j0 + 63; per key tile the CTA gathers those rows of PK
// and PQ into shared memory, computes C1 = Q PKwin^T and C2 = K PQwin^T (64 x 128 each, fp32, shared memory) next to
// S = Q K^T, and adds C1[i][w] + C2[j][w] with w = (i - i0) - (j - j0) + 63 to S before the online softmax.  Single-
// buffered: one cp.async group per key tile.
#include <stdint.h>

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
struct RelCfg {
  static constexpr int kElem = F16 ? 2 : 4;
  static constexpr int kPerChunk = 16 / kElem;
  static constexpr int kLds = F16 ? 72 : 68;
  static constexpr int kTile = BKV * kLds;  // K or V^T tile
  static constexpr int kWin = WIN * kLds;   // PK or PQ window
  static constexpr int kSmem = (2 * kTile + 2 * kWin) * kElem + 2 * BQ * LDC * 4;
};

__device__ __forceinline__ void mma_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// A fragments (16 rows x 64 head dims) of rows lo / hi (row-major, 64 contiguous elements each)
template <bool F16, typename T>
__device__ __forceinline__ void load_a(uint32_t (&a)[F16 ? 4 : 8][4], const T* lo, const T* hi, int t) {
#pragma unroll
  for (int ks = 0; ks < (F16 ? 4 : 8); ++ks) {
    if (F16) {
      const uint32_t* l = reinterpret_cast<const uint32_t*>(lo + ks * 16);
      const uint32_t* h = reinterpret_cast<const uint32_t*>(hi + ks * 16);
      a[ks][0] = l[t]; a[ks][1] = h[t]; a[ks][2] = l[t + 4]; a[ks][3] = h[t + 4];
    } else {
      const uint32_t* l = reinterpret_cast<const uint32_t*>(lo) + ks * 8;
      const uint32_t* h = reinterpret_cast<const uint32_t*>(hi) + ks * 8;
      a[ks][0] = l[t]; a[ks][1] = h[t]; a[ks][2] = l[t + 4]; a[ks][3] = h[t + 4];
    }
  }
}

// c (16 x 8) = A (16 x 64) . B^T for the 8 rows of b starting at b (pitch LDS), then stored to out rows r / r + 8
template <bool F16, typename T, int LDS>
__device__ __forceinline__ void mma_row8(float (&c)[4], const uint32_t (&a)[F16 ? 4 : 8][4], const T* b, int g, int t) {
  c[0] = c[1] = c[2] = c[3] = 0.f;
  const T* br = b + g * LDS;
#pragma unroll
  for (int ks = 0; ks < (F16 ? 4 : 8); ++ks) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(br + ks * (F16 ? 16 : 8));
    if (F16)
      mma_f16(c, a[ks], w[t], w[t + 4]);
    else
      mma_tf32(c, a[ks], w[t], w[t + 4]);
  }
}

// out_mode: 0 fp32, 1 tf32-rounded fp32, 2 bf16 hi | lo split rows, 3 fp16
template <bool F16>
__global__ void __launch_bounds__(THREADS, 1)
disentangled_attention_kernel(const void* __restrict__ qkv_, const void* __restrict__ vt_, long long vt_ld,
                              const void* __restrict__ pk_, const void* __restrict__ pq_, long long pos_ld, int span,
                              const int* __restrict__ rel_row, float scale, void* __restrict__ ctx,
                              const int* __restrict__ cu_seqlens, long long tokens, int max_seqlen, int heads,
                              int out_mode) {
  using Cfg = RelCfg<F16>;
  using T = typename std::conditional<F16, uint16_t, float>::type;
  constexpr int LDS = Cfg::kLds;
  constexpr int KS = F16 ? 4 : 8;
  extern __shared__ __align__(16) uint8_t smem_rel[];
  T* Ks = reinterpret_cast<T*>(smem_rel);  // [BKV][LDS]
  T* Vs = Ks + Cfg::kTile;                 // [HD][LDS]: V^T, keys along the row
  T* PKw = Vs + Cfg::kTile;                // [WIN][LDS]
  T* PQw = PKw + Cfg::kWin;                // [WIN][LDS]
  float* C1 = reinterpret_cast<float*>(PQw + Cfg::kWin);  // [BQ][LDC]: q_i . PKwin[w]
  float* C2 = C1 + BQ * LDC;                               // [BKV][LDC]: k_j . PQwin[w]

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
  const T* pkbase = static_cast<const T*>(pk_) + h * HD;
  const T* pqbase = static_cast<const T*>(pq_) + h * HD;
  const int max_row = 2 * span - 1, max_idx = 2 * max_seqlen - 2;

  uint32_t qa[KS][4];
  load_a<F16>(qa, qbase + (long long)min(q0 + warp * 16 + g, len - 1) * ld,
              qbase + (long long)min(q0 + warp * 16 + g + 8, len - 1) * ld, t);

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
      const int ri = min(max(d0 + w + max_seqlen - 1, 0), max_idx);
      const long long row = min(max(__ldg(rel_row + ri), 0), max_row);
      cp_async16(PKw + w * LDS + c, pkbase + row * pos_ld + c, 16);
      cp_async16(PQw + w * LDS + c, pqbase + row * pos_ld + c, 16);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();

    // ---- S = Q K^T (16 x 64 per warp) ----
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) mma_row8<F16, T, LDS>(s[nt], qa, Ks + nt * 8 * LDS, g, t);
    // ---- C1 = Q PKwin^T (this warp's 16 rows) and C2 = K PQwin^T (keys 16 warp .. 16 warp + 15) ----
    {
      const int r = warp * 16 + g;
#pragma unroll 4
      for (int nt = 0; nt < WIN / 8; ++nt) {
        float c[4];
        mma_row8<F16, T, LDS>(c, qa, PKw + nt * 8 * LDS, g, t);
        *reinterpret_cast<float2*>(C1 + r * LDC + nt * 8 + 2 * t) = make_float2(c[0], c[1]);
        *reinterpret_cast<float2*>(C1 + (r + 8) * LDC + nt * 8 + 2 * t) = make_float2(c[2], c[3]);
      }
      uint32_t ka[KS][4];
      load_a<F16>(ka, Ks + r * LDS, Ks + (r + 8) * LDS, t);
#pragma unroll 4
      for (int nt = 0; nt < WIN / 8; ++nt) {
        float c[4];
        mma_row8<F16, T, LDS>(c, ka, PQw + nt * 8 * LDS, g, t);
        *reinterpret_cast<float2*>(C2 + r * LDC + nt * 8 + 2 * t) = make_float2(c[0], c[1]);
        *reinterpret_cast<float2*>(C2 + (r + 8) * LDC + nt * 8 + 2 * t) = make_float2(c[2], c[3]);
      }
    }
    __syncthreads();
    // ---- S += C1[i][w] + C2[j][w], w = i - j + 63; mask keys outside the sentence ----
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = warp * 16 + g + (e >> 1) * 8, jj = nt * 8 + 2 * t + (e & 1);
        const int w = i - jj + (BKV - 1);
        const int k = rel0 + jj;
        s[nt][e] = (k < 0 || k >= len) ? -INFINITY : s[nt][e] + C1[i * LDC + w] + C2[jj * LDC + w];
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
    __syncthreads();  // everyone is done with the tiles and C1 / C2 before the next key tile overwrites them
  }

  // ---- finalize ----
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
  const float inv_lo = 1.0f / l_lo, inv_hi = 1.0f / l_hi;
  const int row_lo = q0 + warp * 16 + g, row_hi = row_lo + 8;
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
int launch_rel(const void* qkv, const void* vt, long long vt_ld, const void* pos_k, const void* pos_q,
               long long pos_ld, int span, const int32_t* rel_row, float scale, void* ctx, const int32_t* cu_seqlens,
               int n_seq, long long tokens, int max_seqlen, int heads, int out_mode, cudaStream_t stream) {
  using Cfg = RelCfg<F16>;
  static MerPerDevice attr_set;
  if (attr_set.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(disentangled_attention_kernel<F16>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    attr_set.mark();
  }
  dim3 grid((max_seqlen + BQ - 1) / BQ, heads, n_seq);
  disentangled_attention_kernel<F16><<<grid, THREADS, Cfg::kSmem, stream>>>(
      qkv, vt, vt_ld, pos_k, pos_q, pos_ld, span, rel_row, scale, ctx, cu_seqlens, tokens, max_seqlen, heads,
      out_mode);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" int mer_disentangled_attention(const void* qkv, const void* vt, long long vt_ld, const void* pos_k,
                                          const void* pos_q, long long pos_ld, int span, const int32_t* rel_row,
                                          float scale, void* ctx, const int32_t* cu_seqlens, int n_seq,
                                          long long tokens, int max_seqlen, int heads, int flags, void* stream_) {
  const char* name = "mer_disentangled_attention";
  const bool f16 = (flags & MER_ATT_QKV_F16) != 0;
  const int out_flags = flags & ~MER_ATT_QKV_F16;
  MER_REQUIRE(out_flags == 0 || out_flags == MER_EPI_ROUND_TF32 || out_flags == MER_EPI_SPLIT_BF16 ||
                  out_flags == MER_EPI_OUT_F16,
              "%s: flags %d (MER_ATT_QKV_F16 and at most one of MER_EPI_ROUND_TF32 / MER_EPI_SPLIT_BF16 / "
              "MER_EPI_OUT_F16)", name, flags);
  MER_REQUIRE(qkv && vt && ctx && cu_seqlens, "%s: null operand", name);
  MER_REQUIRE(pos_k && pos_q && rel_row, "%s: null relative-position table (pos_k, pos_q or rel_row)", name);
  MER_REQUIRE(heads > 0 && heads <= 65535, "%s: heads %d (1 .. 65535)", name, heads);
  MER_REQUIRE(n_seq > 0 && n_seq <= 65535, "%s: n_seq %d (1 .. 65535)", name, n_seq);
  MER_REQUIRE(span > 0, "%s: span %d (the tables have 2 span > 0 rows)", name, span);
  const int per_chunk = f16 ? 8 : 4;
  MER_REQUIRE(vt_ld >= tokens && vt_ld % per_chunk == 0, "%s: V^T pitch %lld must be a multiple of %d >= tokens %lld",
              name, vt_ld, per_chunk, tokens);
  MER_REQUIRE(pos_ld >= (long long)heads * HD && pos_ld % per_chunk == 0,
              "%s: table pitch %lld must be a multiple of %d >= heads * 64", name, pos_ld, per_chunk);
  MER_REQUIRE(aligned16(qkv) && aligned16(vt) && aligned16(pos_k) && aligned16(pos_q),
              "%s: qkv, vt, pos_k and pos_q must be 16-byte aligned", name);
  MER_REQUIRE(max_seqlen > 0 && max_seqlen <= tokens, "%s: max_seqlen %d (1 .. tokens %lld)", name, max_seqlen,
              tokens);
  const int out_mode = out_flags == MER_EPI_OUT_F16 ? 3 : out_flags == MER_EPI_SPLIT_BF16 ? 2
                       : out_flags == MER_EPI_ROUND_TF32 ? 1 : 0;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (f16)
    return launch_rel<true>(qkv, vt, vt_ld, pos_k, pos_q, pos_ld, span, rel_row, scale, ctx, cu_seqlens, n_seq,
                            tokens, max_seqlen, heads, out_mode, stream);
  return launch_rel<false>(qkv, vt, vt_ld, pos_k, pos_q, pos_ld, span, rel_row, scale, ctx, cu_seqlens, n_seq, tokens,
                           max_seqlen, heads, out_mode, stream);
}
