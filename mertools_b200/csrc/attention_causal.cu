// attention_causal.cu — causal softmax(Q K^T / sqrt(128)) V for packed variable-length sequences with head_dim 128:
// the self-attention of HF LlamaAttention (eager / sdpa, is_causal) as the LLaMA text extractor runs it
// (extract_text_huggingface.py:170-196 -> mertools_b200/extract/llama_text.py).
//
// Operands follow the fp16 V^T kernel of attention_f16.cu: q | k as fp16 rows of the QKV GEMM output
// ([tokens, 3 * heads * 128], rotary embedding already applied by mer_rope_f16, V columns unused), V^T as the GEMM's
// fp16 transposed side output ([heads * 128, vt_ld], vt[d, token]); ctx is written as fp16 rows for the fp16 o_proj
// GEMM.  Flash-style: one CTA = (64-query block, head, sequence), 4 warps x 16 query rows, S = Q K^T and O += P V on
// mma.sync.m16n8k16 (fp16 in, fp32 accumulate), P rounded to fp16, online-softmax statistics in fp32 registers.
// K [64 keys][128 d] and V^T [128 d][64 keys] tiles are double-buffered in shared memory by cp.async.
//
// Causal work: a query block stops at the key tile holding its last row; only tiles that cross the diagonal (or the
// sequence start) are masked, and a warp whose 16 rows all lie before a tile skips that tile's MMAs.  Query blocks are
// issued longest-first.  The key axis begins at the sequence start rounded down to 8 tokens (16-byte copies), so the
// up to 7 leading foreign keys are masked; keys beyond `tokens` are zero-filled, so that masked probabilities (exactly
// 0) never meet V^T padding.  No length cap: the host bounds sequences by max_position_embeddings.
#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int HD = 128;
constexpr int BQ = 64;
constexpr int BKV = 64;
constexpr int THREADS = 128;
// padded row pitches (fp16 elements): K rows 68 words, V^T rows 36 words -> conflict-free fragment loads
constexpr int LDK = HD + 8;
constexpr int LDV = BKV + 8;
constexpr int K_TILE = BKV * LDK;
constexpr int V_TILE = HD * LDV;
constexpr int SMEM = 2 * (K_TILE + V_TILE) * 2;

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

__global__ void __launch_bounds__(THREADS, 2)
causal_attention_kernel(const uint16_t* __restrict__ qkv, const uint16_t* __restrict__ vt_, long long vt_ld,
                        uint16_t* __restrict__ ctx, const int* __restrict__ cu_seqlens, long long tokens, int heads) {
  extern __shared__ __align__(16) uint8_t smem_att[];
  uint16_t* Ks = reinterpret_cast<uint16_t*>(smem_att);  // [2][BKV][LDK]
  uint16_t* Vs = Ks + 2 * K_TILE;                         // [2][HD][LDV]: V^T, keys along the row

  const int seq = blockIdx.z, h = blockIdx.y;
  const int start = cu_seqlens[seq];
  const int len = cu_seqlens[seq + 1] - start;
  const int q0 = (gridDim.x - 1 - blockIdx.x) * BQ;  // longest query blocks first
  if (q0 >= len) return;
  const int kstart = start & ~7, shift = start - kstart;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const long long ld = 3ll * heads * HD;
  const uint16_t* qbase = qkv + (long long)start * ld + h * HD;
  const uint16_t* kbase = qkv + heads * HD + h * HD;  // row = absolute token index
  const uint16_t* vtbase = vt_ + (long long)h * HD * vt_ld;

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
    uint16_t* kd = Ks + buf * K_TILE;
    uint16_t* vd = Vs + buf * V_TILE;
#pragma unroll
    for (int i = 0; i < BKV * (HD / 8) / THREADS; ++i) {  // K: 64 rows x 16 chunks
      const int idx = tid + i * THREADS;
      const int r = idx >> 4, c = (idx & 15) * 8;
      const int key = p0 + r;
      const bool kin = key >= start && key < start + len;
      cp_async16(kd + r * LDK + c, kbase + (long long)(kin ? key : start) * ld + c, kin ? 16 : 0);
    }
#pragma unroll
    for (int i = 0; i < HD * (BKV / 8) / THREADS; ++i) {  // V^T: 128 rows x 8 chunks
      const int idx = tid + i * THREADS;
      const int r = idx >> 3, c = (idx & 7) * 8;
      const long long vk = p0 + c;
      const int vbytes = vk >= tokens ? 0 : (int)min(16ll, (tokens - vk) * 2);
      cp_async16(vd + r * LDV + c, vtbase + (long long)r * vt_ld + (vbytes ? vk : 0), vbytes);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  load_tile(0, 0);
  constexpr float SL2 = 0.08838834764831845f * 1.4426950408889634f;  // 1/sqrt(128) * log2(e)

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
      const uint16_t* kt = Ks + buf * K_TILE;
      const uint16_t* vt = Vs + buf * V_TILE;
      float s[BKV / 8][4];
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(kt + (nt * 8 + g) * LDK);
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks) mma_f16(s[nt], qa[ks], w[ks * 8 + t], w[ks * 8 + t + 4]);
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

}  // namespace

extern "C" int mer_causal_attention_f16(const void* qkv16, const void* vt16, long long vt_ld, void* ctx16,
                                        const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen,
                                        int heads, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(qkv16 && vt16 && ctx16 && cu_seqlens, "mer_causal_attention_f16: null operand");
  MER_REQUIRE(vt_ld >= tokens && vt_ld % 8 == 0, "mer_causal_attention_f16: V^T pitch %lld must be a multiple of 8 >= tokens",
              vt_ld);
  MER_REQUIRE(max_seqlen > 0 && max_seqlen <= tokens, "mer_causal_attention_f16: max_seqlen %d (1 .. tokens %lld)",
              max_seqlen, tokens);
  MER_REQUIRE(heads > 0 && heads <= 65535 && n_seq > 0 && n_seq <= 65535,
              "mer_causal_attention_f16: bad grid (%d heads, %d seqs)", heads, n_seq);
  static MerPerDevice attr_set;
  if (attr_set.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(causal_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr_set.mark();
  }
  dim3 grid((max_seqlen + BQ - 1) / BQ, heads, n_seq);
  causal_attention_kernel<<<grid, THREADS, SMEM, stream>>>(static_cast<const uint16_t*>(qkv16),
                                                           static_cast<const uint16_t*>(vt16), vt_ld,
                                                           static_cast<uint16_t*>(ctx16), cu_seqlens, tokens, heads);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}
