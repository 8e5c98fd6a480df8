// attention_causal.cu — causal softmax(Q K^T / sqrt(HD)) V for packed variable-length sequences: the self-attention of
// HF LlamaAttention (eager / sdpa, is_causal) as the LLaMA text extractor runs it (extract_text_huggingface.py:170-196
// -> mertools_b200/extract/llama_text.py) and of OPTAttention at head_dim HD = 128, and of GPT2Attention at HD = 64
// (gpt2-chinese-cluecorpussmall) and 96 (Wenzhong2.0-GPT2-3.5B) (mertools_b200/extract/ln_decoder_text.py).  The
// kernel is a template on HD; mer_causal_attention_f16 is the HD = 128 instance, mer_causal_attention_hd_f16 picks one
// of the three at run time.
//
// Operands follow the fp16 V^T kernel of attention_f16.cu: q | k as fp16 rows of the QKV GEMM output
// ([tokens, 3 * heads * HD], rotary embedding already applied by mer_rope_f16 for LLaMA, V columns unused), V^T as the
// GEMM's fp16 transposed side output ([heads * HD, vt_ld], vt[d, token]); ctx is written as fp16 rows for the fp16
// o_proj GEMM.  Flash-style: one CTA = (64-query block, head, sequence), 4 warps x 16 query rows, S = Q K^T and
// O += P V on mma.sync.m16n8k16 (fp16 in, fp32 accumulate), P rounded to fp16, online-softmax statistics in fp32
// registers.  K [64 keys][HD d] and V^T [HD d][64 keys] tiles are double-buffered in shared memory by cp.async.
//
// Causal work: a query block stops at the key tile holding its last row; only tiles that cross the diagonal (or the
// sequence start) are masked, and a warp whose 16 rows all lie before a tile skips that tile's MMAs.  Query blocks are
// issued longest-first.  The key axis begins at the sequence start rounded down to 8 tokens (16-byte copies), so the
// up to 7 leading foreign keys are masked; keys beyond `tokens` are zero-filled, so that masked probabilities (exactly
// 0) never meet V^T padding.  No length cap: the host bounds sequences by max_position_embeddings.
//
// ALiBi variant (template ALIBI = true; HF BloomAttention, mertools_b200/extract/ln_decoder_text.py): the score of query
// i and key j of a sequence is q_i . k_j / sqrt(128) + slope_h * (j - i), formed in fp32 before the row maximum, with i
// and j counted from the sequence start (not the packed position).  HF adds slope_h * j; the per-row constant
// slope_h * i cancels in the softmax, and with (j - i) <= 0 the bias stays bounded however long the row is.  Masked and
// foreign keys stay -inf.  ALIBI = false is the LLaMA kernel, unchanged.  ALiBi is instantiated at HD = 128 only.
//
// Multi-query variant (template MQA = true; HF FalconAttention with multi_query, mertools_b200/extract/ln_decoder_text.py):
// every query head reads the one K head and the one V^T head.  Q is columns [0, heads * HD) of qkv rows of pitch qkv_ld,
// K the next HD columns, V^T is [HD, vt_ld].  Only the row pitch, the K column base and the V^T row base differ from the
// plain kernel; nothing is expanded to `heads` copies.  Instantiated at HD = 64 only.
#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int BQ = 64;
constexpr int BKV = 64;
constexpr int THREADS = 128;
// Padded row pitches (fp16 elements).  A fragment load reads word t of row g (g < 8, t < 4): K rows are (HD + 8) / 2
// words apart, i.e. 36 / 52 / 68 at head_dim 64 / 96 / 128, so the banks are 4g + t, 20g + t and 4g + t (mod 32), 32
// distinct banks in each case; V^T rows are 36 words apart.
template <int HD> constexpr int LDK = HD + 8;
constexpr int LDV = BKV + 8;
template <int HD> constexpr int K_TILE = BKV * LDK<HD>;
template <int HD> constexpr int V_TILE = HD * LDV;
template <int HD> constexpr int SMEM = 2 * (K_TILE<HD> + V_TILE<HD>) * 2;
// log2(e) / sqrt(head_dim): the softmax runs in base 2 with the score scale folded in
template <int HD> constexpr float SCALE_LOG2E =
    (HD == 128 ? 0.08838834764831845f : HD == 96 ? 0.10206207261596575f : 0.125f) * 1.4426950408889634f;

__device__ __forceinline__ void mma_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
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

template <int HD, bool ALIBI, bool MQA>
__global__ void __launch_bounds__(THREADS, 2)
causal_attention_kernel(const uint16_t* __restrict__ qkv, const uint16_t* __restrict__ vt_, long long vt_ld,
                        uint16_t* __restrict__ ctx, const int* __restrict__ cu_seqlens, long long tokens, int heads,
                        const float* __restrict__ slopes, long long qkv_ld) {
  static_assert(HD == 64 || HD == 96 || HD == 128, "head_dim 64, 96 or 128");
  static_assert(!ALIBI || HD == 128, "the ALiBi kernel is head_dim 128 only");
  static_assert(!MQA || (HD == 64 && !ALIBI), "the multi-query kernel is head_dim 64 only, without ALiBi");
  constexpr int LDK_ = LDK<HD>, K_TILE_ = K_TILE<HD>, V_TILE_ = V_TILE<HD>;
  extern __shared__ __align__(16) uint8_t smem_att[];
  uint16_t* Ks = reinterpret_cast<uint16_t*>(smem_att);  // [2][BKV][LDK_]
  uint16_t* Vs = Ks + 2 * K_TILE_;                        // [2][HD][LDV]: V^T, keys along the row

  const int seq = blockIdx.z, h = blockIdx.y;
  const int start = cu_seqlens[seq];
  const int len = cu_seqlens[seq + 1] - start;
  const int q0 = (gridDim.x - 1 - blockIdx.x) * BQ;  // longest query blocks first
  if (q0 >= len) return;
  const int kstart = start & ~7, shift = start - kstart;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const long long ld = MQA ? qkv_ld : 3ll * heads * HD;
  const uint16_t* qbase = qkv + (long long)start * ld + h * HD;
  const uint16_t* kbase = qkv + heads * HD + (MQA ? 0 : h * HD);  // row = absolute token index
  const uint16_t* vtbase = vt_ + (MQA ? 0ll : (long long)h * HD * vt_ld);

  const int row_lo = q0 + warp * 16 + g, row_hi = row_lo + 8;
  // last key each row may see (rows past the sequence end are computed on clamped data and never stored)
  const int lim_lo = min(row_lo, len - 1), lim_hi = min(row_hi, len - 1);
  const int warp_last = min(q0 + warp * 16 + 15, len - 1);

  uint32_t qa[HD / 16][4];
  {
    const uint32_t* lo = reinterpret_cast<const uint32_t*>(qbase + (long long)lim_lo * ld);
    const uint32_t* hi = reinterpret_cast<const uint32_t*>(qbase + (long long)lim_hi * ld);
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      qa[ks][0] = lo[ks * 8 + t]; qa[ks][1] = hi[ks * 8 + t]; qa[ks][2] = lo[ks * 8 + t + 4]; qa[ks][3] = hi[ks * 8 + t + 4];
    }
  }

  float o[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  const int q_last = min(q0 + BQ - 1, len - 1);
  const int n_kv = (q_last + shift) / BKV + 1;  // tiles up to the one holding the block's last row

  auto load_tile = [&](int j, int buf) {
    const int p0 = kstart + j * BKV;  // first key position (absolute token index) of the tile
    uint16_t* kd = Ks + buf * K_TILE_;
    uint16_t* vd = Vs + buf * V_TILE_;
#pragma unroll
    for (int i = 0; i < BKV * (HD / 8) / THREADS; ++i) {  // K: 64 rows x HD / 8 chunks (4 / 6 / 8 per thread)
      const int idx = tid + i * THREADS;
      // chunk -> (row, column); shift and mask where HD / 8 is a power of two
      const int r = HD == 96 ? idx / 12 : idx >> (HD == 128 ? 4 : 3);
      const int c = (HD == 96 ? idx % 12 : idx & (HD / 8 - 1)) * 8;
      const int key = p0 + r;
      const bool kin = key >= start && key < start + len;
      cp_async16(kd + r * LDK_ + c, kbase + (long long)(kin ? key : start) * ld + c, kin ? 16 : 0);
    }
#pragma unroll
    for (int i = 0; i < HD * (BKV / 8) / THREADS; ++i) {  // V^T: HD rows x 8 chunks (4 / 6 / 8 per thread)
      const int idx = tid + i * THREADS;
      const int r = idx >> 3, c = (idx & 7) * 8;
      const long long vk = p0 + c;
      const int vbytes = vk >= tokens ? 0 : (int)min(16ll, (tokens - vk) * 2);
      cp_async16(vd + r * LDV + c, vtbase + (long long)r * vt_ld + (vbytes ? vk : 0), vbytes);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  load_tile(0, 0);
  constexpr float SL2 = SCALE_LOG2E<HD>;
  // ALiBi bias in the units of the raw product q.k (the scale is folded into SL2): slope * sqrt(128) per key step, so
  // that zero slopes leave s, and the output, bit-identical to the plain kernel
  const float slope = ALIBI ? __ldg(slopes + h) * 11.313708498984761f : 0.f;

  for (int j = 0; j < n_kv; ++j) {
    const int buf = j & 1;
    if (j + 1 < n_kv) {
      load_tile(j + 1, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const int rel0 = j * BKV - shift;  // key index inside the sequence of tile column 0
    if (rel0 <= warp_last) {           // otherwise every key of the tile is in this warp's future
      const uint16_t* kt = Ks + buf * K_TILE_;
      const uint16_t* vt = Vs + buf * V_TILE_;
      float s[BKV / 8][4];
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(kt + (nt * 8 + g) * LDK_);
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks) mma_f16(s[nt], qa[ks], w[ks * 8 + t], w[ks * 8 + t + 4]);
      }
      if (ALIBI) {  // s / sqrt(128) = q.k / sqrt(128) + slope_h * (j - i)
#pragma unroll
        for (int nt = 0; nt < BKV / 8; ++nt) {
          const int k0 = rel0 + nt * 8 + 2 * t;
          s[nt][0] = fmaf(slope, (float)(k0 - row_lo), s[nt][0]);
          s[nt][1] = fmaf(slope, (float)(k0 + 1 - row_lo), s[nt][1]);
          s[nt][2] = fmaf(slope, (float)(k0 - row_hi), s[nt][2]);
          s[nt][3] = fmaf(slope, (float)(k0 + 1 - row_hi), s[nt][3]);
        }
      }
      // ---- mask foreign leading keys and keys after the row (diagonal / first tiles only) ----
      if (rel0 < 0 || rel0 + BKV - 1 > q0 + warp * 16) {
#pragma unroll
        for (int nt = 0; nt < BKV / 8; ++nt) {
          const int k0 = rel0 + nt * 8 + 2 * t;
          if (k0 < 0 || k0 > lim_lo) s[nt][0] = -INFINITY;
          if (k0 + 1 < 0 || k0 + 1 > lim_lo) s[nt][1] = -INFINITY;
          if (k0 < 0 || k0 > lim_hi) s[nt][2] = -INFINITY;
          if (k0 + 1 < 0 || k0 + 1 > lim_hi) s[nt][3] = -INFINITY;
        }
      }
      // ---- online softmax (base 2, scale folded in) ----
      float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
        mx_lo = fmaxf(mx_lo, fmaxf(s[nt][0], s[nt][1]));
        mx_hi = fmaxf(mx_hi, fmaxf(s[nt][2], s[nt][3]));
      }
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
      // key 0 of the sequence lies in tile 0 and every row sees it, so m is finite from tile 0 on
      const float mn_lo = fmaxf(m_lo, mx_lo), mn_hi = fmaxf(m_hi, mx_hi);
      const float sc_lo = fast_ex2((m_lo - mn_lo) * SL2), sc_hi = fast_ex2((m_hi - mn_hi) * SL2);
      m_lo = mn_lo;
      m_hi = mn_hi;
      const float b_lo = mn_lo * SL2, b_hi = mn_hi * SL2;
      float ps_lo = 0.f, ps_hi = 0.f;
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
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
      // ---- O += P V: 16 keys per step = n-tiles 2 ks and 2 ks + 1 of S ----
#pragma unroll
      for (int ks = 0; ks < BKV / 16; ++ks) {
        uint32_t pa[4];
        pa[0] = pack_f16x2(s[2 * ks][0], s[2 * ks][1]);
        pa[1] = pack_f16x2(s[2 * ks][2], s[2 * ks][3]);
        pa[2] = pack_f16x2(s[2 * ks + 1][0], s[2 * ks + 1][1]);
        pa[3] = pack_f16x2(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
        for (int dt = 0; dt < HD / 8; ++dt) {
          const uint32_t* w = reinterpret_cast<const uint32_t*>(vt + (dt * 8 + g) * LDV + ks * 16);
          mma_f16(o[dt], pa, w[t], w[t + 4]);
        }
      }
    }
    __syncthreads();  // everyone is done with buf before the next prefetch overwrites it
  }

  // ---- finalize: fp16 ctx rows ----
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
  const float inv_lo = 1.0f / l_lo, inv_hi = 1.0f / l_hi;
  const long long ldc = (long long)heads * HD;
  uint16_t* c_lo = ctx + (long long)(start + row_lo) * ldc + h * HD + 2 * t;
  uint16_t* c_hi = ctx + (long long)(start + row_hi) * ldc + h * HD + 2 * t;
#pragma unroll
  for (int dt = 0; dt < HD / 8; ++dt) {
    if (row_lo < len) *reinterpret_cast<uint32_t*>(c_lo + dt * 8) = pack_f16x2(o[dt][0] * inv_lo, o[dt][1] * inv_lo);
    if (row_hi < len) *reinterpret_cast<uint32_t*>(c_hi + dt * 8) = pack_f16x2(o[dt][2] * inv_hi, o[dt][3] * inv_hi);
  }
}

template <int HD, bool ALIBI, bool MQA = false>
int launch_causal(const char* name, const void* qkv16, const void* vt16, long long vt_ld, void* ctx16,
                  const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen, int heads,
                  const float* slopes, cudaStream_t stream, long long qkv_ld = 0) {
  MER_REQUIRE(qkv16 && vt16 && ctx16 && cu_seqlens, "%s: null operand", name);
  MER_REQUIRE(vt_ld >= tokens && vt_ld % 8 == 0, "%s: V^T pitch %lld must be a multiple of 8 >= tokens", name, vt_ld);
  MER_REQUIRE(max_seqlen > 0 && max_seqlen <= tokens, "%s: max_seqlen %d (1 .. tokens %lld)", name, max_seqlen, tokens);
  MER_REQUIRE(heads > 0 && heads <= 65535 && n_seq > 0 && n_seq <= 65535, "%s: bad grid (%d heads, %d seqs)", name,
              heads, n_seq);
  static MerPerDevice attr_set;
  if (attr_set.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(causal_attention_kernel<HD, ALIBI, MQA>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM<HD>));
    attr_set.mark();
  }
  dim3 grid((max_seqlen + BQ - 1) / BQ, heads, n_seq);
  causal_attention_kernel<HD, ALIBI, MQA><<<grid, THREADS, SMEM<HD>, stream>>>(
      static_cast<const uint16_t*>(qkv16), static_cast<const uint16_t*>(vt16), vt_ld, static_cast<uint16_t*>(ctx16),
      cu_seqlens, tokens, heads, slopes, qkv_ld);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}

}  // namespace

extern "C" int mer_causal_attention_f16(const void* qkv16, const void* vt16, long long vt_ld, void* ctx16,
                                        const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen,
                                        int heads, void* stream_) {
  return launch_causal<128, false>("mer_causal_attention_f16", qkv16, vt16, vt_ld, ctx16, cu_seqlens, n_seq, tokens,
                                   max_seqlen, heads, nullptr, static_cast<cudaStream_t>(stream_));
}

extern "C" int mer_causal_alibi_attention_f16(const void* qkv16, const void* vt16, long long vt_ld, void* ctx16,
                                              const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen,
                                              int heads, const float* slopes, void* stream_) {
  MER_REQUIRE(slopes, "mer_causal_alibi_attention_f16: null slopes");
  return launch_causal<128, true>("mer_causal_alibi_attention_f16", qkv16, vt16, vt_ld, ctx16, cu_seqlens, n_seq,
                                  tokens, max_seqlen, heads, slopes, static_cast<cudaStream_t>(stream_));
}

extern "C" int mer_causal_attention_hd_f16(const void* qkv16, const void* vt16, long long vt_ld, void* ctx16,
                                           const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen,
                                           int heads, int head_dim, void* stream_) {
  const char* name = "mer_causal_attention_hd_f16";
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(head_dim == 64 || head_dim == 96 || head_dim == 128, "%s: head_dim %d (64, 96 or 128)", name, head_dim);
  switch (head_dim) {
    case 64:
      return launch_causal<64, false>(name, qkv16, vt16, vt_ld, ctx16, cu_seqlens, n_seq, tokens, max_seqlen, heads,
                                      nullptr, stream);
    case 96:
      return launch_causal<96, false>(name, qkv16, vt16, vt_ld, ctx16, cu_seqlens, n_seq, tokens, max_seqlen, heads,
                                      nullptr, stream);
    default:
      return launch_causal<128, false>(name, qkv16, vt16, vt_ld, ctx16, cu_seqlens, n_seq, tokens, max_seqlen, heads,
                                       nullptr, stream);
  }
}

extern "C" int mer_causal_mqa_attention_f16(const void* qkv16, long long qkv_ld, const void* vt16, long long vt_ld,
                                            void* ctx16, const int32_t* cu_seqlens, int n_seq, long long tokens,
                                            int max_seqlen, int heads, void* stream_) {
  const char* name = "mer_causal_mqa_attention_f16";
  MER_REQUIRE(heads > 0 && heads <= 65535, "%s: %d heads (1 .. 65535)", name, heads);
  MER_REQUIRE(qkv_ld >= (heads + 1ll) * 64 && qkv_ld % 8 == 0,
              "%s: qkv pitch %lld must be a multiple of 8 >= (heads + 1) * 64 = %lld", name, qkv_ld, (heads + 1ll) * 64);
  return launch_causal<64, false, true>(name, qkv16, vt16, vt_ld, ctx16, cu_seqlens, n_seq, tokens, max_seqlen, heads,
                                        nullptr, static_cast<cudaStream_t>(stream_), qkv_ld);
}
