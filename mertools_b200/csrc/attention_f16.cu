// attention_f16.cu — softmax(Q K^T / 8) V for packed variable-length sequences (head_dim 64) that reads V
// transposed: the form the QKV GEMM epilogue writes (V^T [heads*64, vt_ld], vt[d, token], keys contiguous).
// mer_attention_hd runs the same kernel at head_dim 32 and with the score scale as an argument (ALBERT).
//
// Two operand formats share one flash-style kernel:
//   fp16 : q | k fp16 rows of qkv16, fp16 V^T; S = Q K^T and O += P V on mma.sync.m16n8k16 (fp16 in, fp32
//          accumulate), P rounded to fp16.  The ViT / HuBERT / BERT stacks in MER_GEMM_F16 mode and the
//          250 .. 505-token rows of the TF32 / BF16X3 stacks (fp16 carries the same 10 mantissa bits as tf32).
//   tf32 : tf32-rounded fp32 q | k rows and V^T; mma.sync.m16n8k8 tf32, P rounded to tf32.  The TF32 / BF16X3
//          stacks for sequences of up to 253 tokens.
// Replaces the same reference op as attention.cu (HF eager/sdpa attention, modeling_vit.py:171-196,
// modeling_hubert.py:262-345).
//
// One CTA = (64-query block, head, sequence); 4 warps x 16 query rows; K [64 keys][64 d] and V^T [64 d][64 keys]
// tiles double-buffered in shared memory by cp.async; online softmax in fp32 registers.  The S accumulator
// fragment is the A fragment of P V (fp16: two 8-key n-tiles form one 16-key k-step; tf32: keys 2t / 2t+1 of an
// 8-key group are k-columns t / t+4, and the V^T columns are read under the same permutation).
// 16-byte copies need 16-byte aligned starts: the key axis of a sequence begins at its start rounded down to a
// multiple of 8 tokens, and the (up to 7) leading foreign keys are masked.  Keys beyond the last token are
// zero-filled, so that masked probabilities (exactly 0) never meet uninitialised V^T padding.
#include <stdlib.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int BQ = 64;
constexpr int BKV = 64;
constexpr int THREADS = 128;
constexpr int MAX_SEQ = 505;  // longest sequence the stacks send here (10 s audio rows, CLIP L/14)
constexpr int MAX_SEQ_HD = 512;  // mer_attention_hd: ALBERT's position table
// whole-clip audio rows (MER2023's extractor: a 60 s clip is 2,999 HuBERT frames); the emulated fp16-P readout error is
// measured up to this length (scripts/precision_table_long_audio.py)
constexpr int MAX_SEQ_LONG = MER_ATT_LONG_MAX;

template <bool F16, int HD>
struct AttCfg {
  static constexpr int kElem = F16 ? 2 : 4;
  static constexpr int kPerChunk = 16 / kElem;  // elements per 16-byte copy
  // padded row pitches in elements: conflict-free fragment loads.  K rows (HD wide) are 36 (HD 64) / 20 (HD 32) words
  // apart for fp16 and 68 / 36 for tf32; V^T rows (64 keys wide) are 36 (fp16) / 68 (tf32) words apart at every HD.
  static constexpr int kLdsV = F16 ? 72 : 68;
  static constexpr int kLdsK = HD == 64 ? kLdsV : (F16 ? 40 : 36);
  static constexpr int kTileK = BKV * kLdsK;  // elements of one K tile
  static constexpr int kTileV = HD * kLdsV;   // elements of one V^T tile
  static constexpr int kSmem = 2 * (kTileK + kTileV) * kElem;
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

// scale * log2(e): 1/8 (head_dim 64) as a compile-time constant when the kernel has no scale argument, else the argument
template <typename... S>
__device__ __forceinline__ float score_l2(S... sl2) {
  if constexpr (sizeof...(S) == 0) return 0.125f * 1.4426950408889634f;  // 1/sqrt(64) * log2(e)
  else return (sl2 + ...);
}

// out_mode: 0 fp32, 1 tf32-rounded fp32, 2 bf16 hi | lo split rows, 3 fp16.  sl2: empty (scores scaled by 1/8), or one
// float, scale * log2(e) (mer_attention_hd).  The scale is an empty pack rather than a default argument so that the
// head_dim-64 instances mer_attention runs keep their parameter list and code.
template <bool F16, int HD = 64, typename... S>
__global__ void __launch_bounds__(THREADS, 3)
attention_vt_kernel(const void* __restrict__ qkv_, const void* __restrict__ vt_, long long vt_ld, void* __restrict__ ctx,
                    const int* __restrict__ cu_seqlens, long long tokens, int heads, int out_mode, S... sl2) {
  static_assert(HD == 32 || HD == 64, "head_dim 32 or 64");
  using Cfg = AttCfg<F16, HD>;
  using T = typename std::conditional<F16, uint16_t, float>::type;
  // (V^T rows are Cfg::kLdsV apart: a local constexpr for it reorders the front end's output, and the head_dim-64
  // instances are meant to keep their SASS)
  constexpr int LDS = Cfg::kLdsK;   // K rows
  extern __shared__ __align__(16) uint8_t smem_att[];
  T* Ks = reinterpret_cast<T*>(smem_att);  // [2][BKV][LDS]
  T* Vs = Ks + 2 * Cfg::kTileK;            // [2][HD][Cfg::kLdsV]: V^T, keys along the row

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

  // ---- Q fragments ----
  constexpr int QK_STEPS = F16 ? HD / 16 : HD / 8;  // k-steps over head_dim
  uint32_t qa[QK_STEPS][4];
  {
    const T* q_lo = qbase + (long long)min(q0 + warp * 16 + g, len - 1) * ld;
    const T* q_hi = qbase + (long long)min(q0 + warp * 16 + g + 8, len - 1) * ld;
#pragma unroll
    for (int ks = 0; ks < QK_STEPS; ++ks) {
      if (F16) {
        const uint32_t* lo = reinterpret_cast<const uint32_t*>(q_lo + ks * 16);
        const uint32_t* hi = reinterpret_cast<const uint32_t*>(q_hi + ks * 16);
        qa[ks][0] = lo[t]; qa[ks][1] = hi[t]; qa[ks][2] = lo[t + 4]; qa[ks][3] = hi[t + 4];
      } else {
        const float* lo = reinterpret_cast<const float*>(q_lo) + ks * 8;
        const float* hi = reinterpret_cast<const float*>(q_hi) + ks * 8;
        qa[ks][0] = __float_as_uint(lo[t]); qa[ks][1] = __float_as_uint(hi[t]);
        qa[ks][2] = __float_as_uint(lo[t + 4]); qa[ks][3] = __float_as_uint(hi[t + 4]);
      }
    }
  }

  float o[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  const int n_kv = (shift + len + BKV - 1) / BKV;

  auto load_tile = [&](int j, int buf) {
    const int p0 = kstart + j * BKV;  // first key position (absolute token index) of the tile
    T* kd = Ks + buf * Cfg::kTileK;
    T* vd = Vs + buf * Cfg::kTileV;
    if constexpr (HD == BKV) {
      constexpr int CPR = HD / Cfg::kPerChunk;  // 16-byte chunks per 64-element row
#pragma unroll
      for (int i = 0; i < BKV * CPR / THREADS; ++i) {
        const int idx = tid + i * THREADS;
        const int r = idx / CPR, c = (idx % CPR) * Cfg::kPerChunk;
        // K row r = key p0 + r (zero outside the sequence); V^T row r = head dim r, keys p0 + c ..
        const int key = p0 + r;
        const bool kin = key >= start && key < start + len;
        cp_async16(kd + r * LDS + c, kbase + (long long)(kin ? key : start) * ld + c, kin ? 16 : 0);
        const long long vk = p0 + c;
        const int vbytes = vk >= tokens ? 0 : (int)min(16ll, (tokens - vk) * Cfg::kElem);
        cp_async16(vd + r * Cfg::kLdsV + c, vtbase + (long long)r * vt_ld + (vbytes ? vk : 0), vbytes);
      }
    } else {  // K: BKV rows of HD; V^T: HD rows of BKV keys
      constexpr int CPK = HD / Cfg::kPerChunk, CPV = BKV / Cfg::kPerChunk;
#pragma unroll
      for (int i = 0; i < BKV * CPK / THREADS; ++i) {
        const int idx = tid + i * THREADS;
        const int r = idx / CPK, c = (idx % CPK) * Cfg::kPerChunk;
        const int key = p0 + r;
        const bool kin = key >= start && key < start + len;
        cp_async16(kd + r * LDS + c, kbase + (long long)(kin ? key : start) * ld + c, kin ? 16 : 0);
      }
#pragma unroll
      for (int i = 0; i < HD * CPV / THREADS; ++i) {
        const int idx = tid + i * THREADS;
        const int r = idx / CPV, c = (idx % CPV) * Cfg::kPerChunk;
        const long long vk = p0 + c;
        const int vbytes = vk >= tokens ? 0 : (int)min(16ll, (tokens - vk) * Cfg::kElem);
        cp_async16(vd + r * Cfg::kLdsV + c, vtbase + (long long)r * vt_ld + (vbytes ? vk : 0), vbytes);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  load_tile(0, 0);
  const float SL2 = score_l2(sl2...);  // scale * log2(e)

  for (int j = 0; j < n_kv; ++j) {
    const int buf = j & 1;
    if (j + 1 < n_kv) {
      load_tile(j + 1, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const T* kt = Ks + buf * Cfg::kTileK;
    const T* vt = Vs + buf * Cfg::kTileV;

    // ---- S = Q K^T: 16 x 64 per warp ----
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      const T* kr = kt + (nt * 8 + g) * LDS;
#pragma unroll
      for (int ks = 0; ks < QK_STEPS; ++ks) {
        if (F16) {
          const uint32_t* w = reinterpret_cast<const uint32_t*>(kr + ks * 16);
          mma_f16(s[nt], qa[ks], w[t], w[t + 4]);
        } else {
          const uint32_t* w = reinterpret_cast<const uint32_t*>(kr) + ks * 8;
          mma_tf32(s[nt], qa[ks], w[t], w[t + 4]);
        }
      }
    }
    // ---- mask keys outside [start, start + len) (first and last tiles only) ----
    const int rel0 = j * BKV - shift;  // key index inside the sequence of tile column 0
    if (rel0 < 0 || rel0 + BKV > len) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int k0 = rel0 + nt * 8 + 2 * t;
        if (k0 < 0 || k0 >= len) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
        if (k0 + 1 < 0 || k0 + 1 >= len) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
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
    for (int dt = 0; dt < HD / 8; ++dt) {
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
        for (int dt = 0; dt < HD / 8; ++dt) {
          const uint32_t* w = reinterpret_cast<const uint32_t*>(vt + (dt * 8 + g) * Cfg::kLdsV + ks * 16);
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
        for (int dt = 0; dt < HD / 8; ++dt) {
          const float2 w = *reinterpret_cast<const float2*>(
              reinterpret_cast<const float*>(vt) + (dt * 8 + g) * Cfg::kLdsV + ks * 8 + 2 * t);
          mma_tf32(o[dt], pa, __float_as_uint(w.x), __float_as_uint(w.y));
        }
      }
    }
    __syncthreads();  // everyone is done with buf before the next prefetch overwrites it
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
  for (int dt = 0; dt < HD / 8; ++dt) {
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

// max_cap: the longest row the caller routes here (MAX_SEQ for mer_attention, MAX_SEQ_HD for mer_attention_hd; the
// kernel itself loops over any number of 64-key tiles).  scale is read by the RT_SCALE instances only.
template <bool F16, int HD = 64, bool RT_SCALE = false>
int launch_vt(const void* qkv, const void* vt, long long vt_ld, void* ctx, const int* cu_seqlens, int n_seq,
              long long tokens, int heads, int max_seqlen, int out_mode, cudaStream_t stream, int max_cap = MAX_SEQ,
              float scale = 0.125f) {
  MER_REQUIRE(qkv && vt && ctx && cu_seqlens, "mer_attention (V^T): null operand");
  MER_REQUIRE(out_mode >= 0 && out_mode <= 3, "mer_attention (V^T): out_mode %d", out_mode);
  using Cfg = AttCfg<F16, HD>;
  MER_REQUIRE(vt_ld >= tokens && vt_ld % Cfg::kPerChunk == 0,
              "mer_attention (V^T): V^T pitch %lld must be a multiple of %d >= tokens", vt_ld, Cfg::kPerChunk);
  MER_REQUIRE(max_seqlen > 0 && max_seqlen <= max_cap, "mer_attention (V^T): max_seqlen %d (1 .. %d)", max_seqlen,
              max_cap);
  MER_REQUIRE(heads > 0 && heads <= 65535 && n_seq <= 65535, "mer_attention (V^T): bad grid (%d heads, %d seqs)",
              heads, n_seq);
  if (n_seq <= 0 || tokens <= 0) return 0;
  static MerPerDevice attr_set;
  if (attr_set.needs_setup()) {
    if constexpr (RT_SCALE)
      MER_CUDA_CHECK(cudaFuncSetAttribute(attention_vt_kernel<F16, HD, float>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    else
      MER_CUDA_CHECK(cudaFuncSetAttribute(attention_vt_kernel<F16, HD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          Cfg::kSmem));
    attr_set.mark();
  }
  const double s_avg = (double)tokens / n_seq;  // exact for equal-length batches (ViT frames)
  const int prof = mer_prof_begin(F16 ? MER_PROF_ATT_F16 : MER_PROF_ATT_TC,
                                  4.0 * s_avg * s_avg * HD * (double)n_seq * heads, stream);
  dim3 grid((max_seqlen + BQ - 1) / BQ, heads, n_seq);
  if constexpr (RT_SCALE)
    attention_vt_kernel<F16, HD, float><<<grid, THREADS, Cfg::kSmem, stream>>>(
        qkv, vt, vt_ld, ctx, cu_seqlens, tokens, heads, out_mode, scale * 1.4426950408889634f);
  else
    attention_vt_kernel<F16, HD><<<grid, THREADS, Cfg::kSmem, stream>>>(qkv, vt, vt_ld, ctx, cu_seqlens, tokens, heads,
                                                                        out_mode);
  mer_prof_end(prof, stream);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

}  // namespace

// fp16 q | k | V^T for every sequence of up to 505 tokens; MER_ATT_F16_LONG=0 sends rows of 250 .. 505 tokens of the
// TF32 / BF16X3 stacks to the fp32-operand kernel of attention.cu instead (A/B runs)
bool mer_attention_f16_supported(int max_seqlen) {
  if (max_seqlen <= 0 || mer_attention_legacy()) return false;
  if (max_seqlen <= 249) return true;
  const char* e = getenv("MER_ATT_F16_LONG");
  return (e == nullptr || atoi(e) != 0) && max_seqlen <= MAX_SEQ;
}

// rows of 506 .. MAX_SEQ_LONG tokens: the HuBERT / wav2vec2 stacks (MerStackArgs::long_rows), not mer_attention
bool mer_attention_f16_long_supported(int max_seqlen) {
  return max_seqlen > MAX_SEQ && max_seqlen <= MAX_SEQ_LONG && !mer_attention_legacy();
}

int mer_attention_f16_long_launch(const void* qkv16, const void* vt16, long long vt_ld, void* ctx, const int* cu_seqlens,
                                  int n_seq, long long tokens, int heads, int max_seqlen, int out_mode,
                                  cudaStream_t stream) {
  if (max_seqlen <= MAX_SEQ)
    return mer_attention_f16_launch(qkv16, vt16, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode,
                                    stream);
  return launch_vt<true>(qkv16, vt16, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode, stream,
                         MAX_SEQ_LONG);
}

// qkv16: fp16 [tokens, 3*heads*64] (V columns unused), vt16: fp16 [heads*64, vt_ld] with vt[d, token];
// ctx [tokens, heads*64] in the format `out_mode` names (3 fp16, 2 bf16 hi | lo split rows, 1 tf32-rounded fp32, 0 fp32).
// Rows of 129 .. 208 tokens take the one-CTA-per-(sequence, head) kernel of attention_short.cu
// (mer_attention_short_enabled; MER_ATT_SHORT=1: every row of up to 249 tokens).
int mer_attention_f16_launch(const void* qkv16, const void* vt16, long long vt_ld, void* ctx, const int* cu_seqlens,
                             int n_seq, long long tokens, int heads, int max_seqlen, int out_mode, cudaStream_t stream) {
  if (mer_attention_short_enabled(max_seqlen))
    return mer_attention_short_launch(qkv16, vt16, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode,
                                      stream);
  return launch_vt<true>(qkv16, vt16, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode, stream);
}

// tf32-rounded fp32 q | k rows and V^T (the V columns of qkv are not written when V^T is)
int mer_attention_tc_launch(const float* qkv, const float* vt, long long vt_ld, float* ctx, const int* cu_seqlens,
                            int n_seq, long long tokens, int heads, int max_seqlen, int out_mode, cudaStream_t stream) {
  return launch_vt<false>(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode, stream);
}

// mer_attention's V^T route at head_dim 32 or 64 with an explicit score scale (ALBERT: 1 / sqrt(hidden / heads), also
// for heads zero-padded from 26 to 32 columns).  head_dim 64 at scale 1/8 runs exactly what mer_attention runs (the
// kernel of attention_short.cu for fp16 rows of up to 249 tokens, then the compile-time-scale instances); every other
// case runs the tiled kernel with the scale as an argument.  Rows up to MAX_SEQ_HD tokens.
extern "C" int mer_attention_hd(const void* qkv, const void* vt, long long vt_ld, void* ctx, const int32_t* cu_seqlens,
                                int n_seq, long long tokens, int max_seqlen, int heads, int head_dim, float scale,
                                int flags, void* stream_) {
  const char* name = "mer_attention_hd";
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(head_dim == 32 || head_dim == 64, "%s: head_dim %d (32 or 64)", name, head_dim);
  MER_REQUIRE(scale > 0.f && scale <= 1.f, "%s: scale %g (0 < scale <= 1)", name, (double)scale);
  MER_REQUIRE(qkv && vt && ctx && cu_seqlens, "%s: null operand", name);
  MER_REQUIRE((flags & ~(MER_ATT_QKV_F16 | MER_EPI_OUT_F16 | MER_EPI_SPLIT_BF16 | MER_EPI_ROUND_TF32)) == 0,
              "%s: flags 0x%x", name, flags);
  const bool f16 = (flags & MER_ATT_QKV_F16) != 0;
  const int chunk = f16 ? 8 : 4;
  MER_REQUIRE(vt_ld >= tokens && vt_ld % chunk == 0, "%s: V^T pitch %lld must be a multiple of %d >= tokens", name,
              vt_ld, chunk);
  MER_REQUIRE(tokens > 0 && max_seqlen > 0 && max_seqlen <= MAX_SEQ_HD && max_seqlen <= tokens,
              "%s: max_seqlen %d (1 .. min(%d, tokens %lld))", name, max_seqlen, MAX_SEQ_HD, tokens);
  MER_REQUIRE(heads > 0 && heads <= 65535 && n_seq > 0 && n_seq <= 65535, "%s: bad grid (%d heads, %d seqs)", name,
              heads, n_seq);
  const int out_mode = (flags & MER_EPI_OUT_F16) ? 3 : (flags & MER_EPI_SPLIT_BF16) ? 2 : ((flags & MER_EPI_ROUND_TF32) ? 1 : 0);
  if (head_dim == 64 && scale == 0.125f) {
    if (f16 && max_seqlen <= MAX_SEQ)
      return mer_attention_f16_launch(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode,
                                      stream);
    return f16 ? launch_vt<true>(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode, stream,
                                 MAX_SEQ_HD)
               : launch_vt<false>(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode, stream,
                                  MAX_SEQ_HD);
  }
#define MER_ATT_HD(F, H)                                                                                           \
  return launch_vt<F, H, true>(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode, stream, \
                               MAX_SEQ_HD, scale)
  if (head_dim == 32) {
    if (f16) MER_ATT_HD(true, 32);
    MER_ATT_HD(false, 32);
  }
  if (f16) MER_ATT_HD(true, 64);
  MER_ATT_HD(false, 64);
#undef MER_ATT_HD
}

// the fp16 route of mer_attention for rows of up to MAX_SEQ_LONG tokens (mer_b200.h)
extern "C" int mer_attention_long(const void* qkv, const void* vt, long long vt_ld, void* ctx, const int32_t* cu_seqlens,
                                  int n_seq, long long tokens, int max_seqlen, int heads, int flags, void* stream) {
  const char* name = "mer_attention_long";
  MER_REQUIRE(qkv && vt && ctx && cu_seqlens, "%s: null operand", name);
  MER_REQUIRE((flags & ~(MER_EPI_OUT_F16 | MER_EPI_SPLIT_BF16 | MER_EPI_ROUND_TF32)) == 0, "%s: flags 0x%x", name, flags);
  MER_REQUIRE(tokens > 0 && tokens < (1ll << 31), "%s: tokens %lld (1 .. 2^31 - 1: int32 cu_seqlens)", name, tokens);
  MER_REQUIRE(vt_ld >= tokens && vt_ld % 8 == 0, "%s: V^T pitch %lld must be a multiple of 8 >= tokens %lld", name, vt_ld,
              tokens);
  MER_REQUIRE(max_seqlen > 0 && max_seqlen <= MAX_SEQ_LONG && max_seqlen <= tokens,
              "%s: max_seqlen %d (1 .. min(MER_ATT_LONG_MAX = %d, tokens %lld))", name, max_seqlen, MAX_SEQ_LONG, tokens);
  MER_REQUIRE(heads > 0 && heads <= 65535 && n_seq > 0 && n_seq <= 65535, "%s: bad grid (%d heads, %d seqs)", name,
              heads, n_seq);
  const int out_mode = (flags & MER_EPI_OUT_F16) ? 3 : (flags & MER_EPI_SPLIT_BF16) ? 2 : ((flags & MER_EPI_ROUND_TF32) ? 1 : 0);
  return mer_attention_f16_long_launch(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode,
                                       static_cast<cudaStream_t>(stream));
}
