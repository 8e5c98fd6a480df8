// attention_short.cu — softmax(Q K^T / 8) V for packed variable-length fp16 sequences of up to 249 tokens (head_dim
// 64).  Same operands as the fp16 form of attention_f16.cu (q | k fp16 rows of qkv16, fp16 V^T [heads*64, vt_ld]
// written by the QKV GEMM epilogue), same numerics (fp32 scores, scale and log2(e) folded into one FMA before
// ex2.approx, P rounded to fp16, fp32 row statistics, normalisation applied to O), every ctx format (fp16, fp32,
// tf32-rounded fp32, bf16 hi | lo split rows).  mer_attention_short_enabled says which batches come here.
//
// One CTA = one (sequence, head): K and V^T of the pair are loaded once (cp.async) into 128B-swizzled shared memory
// and read with ldmatrix.  16-byte copies need 16-byte aligned starts, so key position p holds token
// (start & ~7) + p; the up to 7 leading foreign keys and the tail of the last 16-key step are masked to -inf.  Keys
// past the last token are zero-filled: masked probabilities (exactly 0) never meet uninitialised V^T padding.
//
// 4 warps loop over the 16-row query slices of the sequence; each slice's Q (2 KB) goes to the warp's own slot,
// which then stages the fp16 ctx slice on the way out (whole 128-byte rows).  Keys run in 16-key steps: a 197-token
// frame computes 208 x (at most 208) scores instead of the tile kernel's 256 x 256.  Up to 128 key positions the
// softmax is exact (all scores in registers); longer rows take two 128-key chunks with one online rescale.
// ~66 KB (197 tokens) to ~73 KB (249) of shared memory and 167 registers: 3 CTAs per SM.
#include <stdlib.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int HD = 64;
constexpr int THREADS = 128;
constexpr int WARPS = THREADS / 32;
constexpr int MAX_SEQ = 249;   // longest row: its keys, shifted by up to 7, fill 256 key positions
constexpr int KPOS_MAX = 256;
constexpr int CHUNK = 128;                // keys per register-resident score chunk
constexpr int ROW_BYTES = HD * 2;         // one fp16 row of 64: one 128-byte swizzle row
constexpr int VBOX_KEYS = 64;             // V^T tile: 64 dims x 64 key positions (one 128-byte swizzle row each)
constexpr int VBOX_BYTES = HD * VBOX_KEYS * 2;
constexpr int QSLOT_BYTES = 16 * ROW_BYTES;  // per warp: 16 query rows

// shared memory of a launch whose longest sequence pads to `kpad` keys (multiple of 16)
constexpr int smem_bytes(int kpad) {
  return 1024 /* 1024-byte alignment of the swizzled tiles */ + kpad * ROW_BYTES +
         (kpad + VBOX_KEYS - 1) / VBOX_KEYS * VBOX_BYTES + WARPS * QSLOT_BYTES;
}

// byte offset of 16-byte chunk `c` of row `r` in a 128B-swizzled tile (1024-byte aligned): conflict-free ldmatrix
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * ROW_BYTES + ((c ^ (r & 7)) << 4)); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void stsm_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}
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

// out_mode: 0 fp32, 1 tf32-rounded fp32, 2 bf16 hi | lo split rows, 3 fp16.
__global__ void __launch_bounds__(THREADS, 3)
attention_short_kernel(const uint16_t* __restrict__ qkv, const uint16_t* __restrict__ vt, long long vt_ld,
                       long long tokens, void* __restrict__ ctx, const int* __restrict__ cu_seqlens, int heads, int kcap,
                       int out_mode) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by offset (as in gemm.cu), so that everything derived from it stays in the shared space
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int n_vbox_cap = (kcap + VBOX_KEYS - 1) / VBOX_KEYS;
  uint8_t* Ks = smem;                                        // [kcap key positions][64 d], swizzled
  uint8_t* Vs = Ks + kcap * ROW_BYTES;                       // [box][64 d][64 key positions], swizzled
  uint8_t* Qs = Vs + n_vbox_cap * VBOX_BYTES;                // [warp][16 rows][64 d], swizzled

  const int h = blockIdx.x, seq = blockIdx.y;
  const int start = cu_seqlens[seq];
  const int len = cu_seqlens[seq + 1] - start;
  // key position p holds token kstart + p: 16-byte copies of V^T need 16-byte aligned starts
  const int kstart = start & ~7, shift = start - kstart, npos = shift + len;
  if (len <= 0) return;
  if (npos > kcap) return;  // a row longer than max_seqlen: the tiles would not fit (ctx rows stay unwritten)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int n16 = (len + 15) >> 4;          // 16-row query slices
  const int nk16 = (npos + 15) >> 4;        // 16-key steps
  const int n_chunks = (nk16 + 7) >> 3;     // 128-key chunks (1 or 2)
  const int ld = 3 * heads * HD;
  uint8_t* qslot = Qs + warp * QSLOT_BYTES;

  // ---- K rows and V^T columns of key positions [0, 16 nk16), once per (sequence, head) ----
  {
    const uint16_t* kbase = qkv + (heads + h) * HD;
    for (int i = tid; i < nk16 * 16 * 8; i += THREADS) {
      const int p = i >> 3, ch = i & 7;
      const long long tok = kstart + p;
      cp_async16(Ks + swz(p, ch), kbase + (tok < tokens ? tok : 0) * ld + ch * 8, tok < tokens ? 16 : 0);
    }
    const uint16_t* vbase = vt + (long long)h * HD * vt_ld;
    const int kch = nk16 * 2;  // 8-key chunks per V^T row
    for (int i = tid; i < HD * kch; i += THREADS) {
      const int d = i / kch, kc = i - d * kch;
      const long long key0 = kstart + kc * 8;
      // keys past the last token are zero-filled: masked probabilities never meet uninitialised padding
      const int bytes = key0 >= tokens ? 0 : (int)min(16ll, (tokens - key0) * 2);
      cp_async16(Vs + (kc >> 3) * VBOX_BYTES + swz(d, kc & 7), vbase + d * vt_ld + (bytes ? key0 : 0), bytes);
    }
  }

  const uint32_t ks_u = smem_u32(Ks), vs_u = smem_u32(Vs);
  const uint32_t qs_u = smem_u32(qslot);
  constexpr float SL2 = 0.125f * 1.4426950408889634f;  // 1/sqrt(64) * log2(e)
  const int ldc = heads * HD;

  // Q rows of a 16-row query slice into the warp's slot
  auto load_q = [&](int sl) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = i * 32 + lane, r = idx >> 3, ch = idx & 7;
      const int tok = start + sl * 16 + r;
      cp_async16(qslot + swz(r, ch), qkv + (long long)(tok < tokens ? tok : 0) * ld + h * HD + ch * 8,
                 tok < tokens ? 16 : 0);
    }
  };
  if (warp < n16) load_q(warp);
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  for (int sl = warp; sl < n16; sl += WARPS) {
    if (sl != warp) {
      load_q(sl);
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncwarp();
    }
    uint32_t qa[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      ldsm_x4(qs_u + swz(lane & 15, 2 * ks + (lane >> 4)), qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3]);

    float o[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;

    for (int c = 0; c < n_chunks; ++c) {
      const int kn = min(8, nk16 - c * 8);  // 16-key steps in this chunk
      // ---- S = Q K^T: 16 x (16 kn) ----
      float s[16][4];
#pragma unroll
      for (int nt = 0; nt < 16; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
        if (nt < 2 * kn) {
          const int key = c * CHUNK + nt * 8 + (lane & 7);
#pragma unroll
          for (int p = 0; p < 2; ++p) {
            uint32_t b0, b1, b2, b3;
            ldsm_x4(ks_u + swz(key, 4 * p + (lane >> 3)), b0, b1, b2, b3);
            mma_f16(s[nt], qa[2 * p], b0, b1);
            mma_f16(s[nt], qa[2 * p + 1], b2, b3);
          }
        }
      }
      // ---- mask key positions outside [shift, shift + len): up to 7 leading foreign keys, the last step's tail ----
      float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 16; ++nt) {
        if (nt < 2 * kn) {
          const int k0 = c * CHUNK + nt * 8 + 2 * t;
          if (k0 < shift || k0 >= npos) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
          if (k0 + 1 < shift || k0 + 1 >= npos) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
          mx_lo = fmaxf(mx_lo, fmaxf(s[nt][0], s[nt][1]));
          mx_hi = fmaxf(mx_hi, fmaxf(s[nt][2], s[nt][3]));
        }
      }
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
      // key 0 is in chunk 0, so the maximum is finite from the first chunk on; there the rescale is ex2(-inf) = 0
      const float mn_lo = fmaxf(m_lo, mx_lo), mn_hi = fmaxf(m_hi, mx_hi);
      const float sc_lo = fast_ex2((m_lo - mn_lo) * SL2), sc_hi = fast_ex2((m_hi - mn_hi) * SL2);
      m_lo = mn_lo;
      m_hi = mn_hi;
      const float b_lo = mn_lo * SL2, b_hi = mn_hi * SL2;
      float ps_lo = 0.f, ps_hi = 0.f;
#pragma unroll
      for (int nt = 0; nt < 16; ++nt) {
        if (nt < 2 * kn) {
          s[nt][0] = fast_ex2(fmaf(s[nt][0], SL2, -b_lo));
          s[nt][1] = fast_ex2(fmaf(s[nt][1], SL2, -b_lo));
          s[nt][2] = fast_ex2(fmaf(s[nt][2], SL2, -b_hi));
          s[nt][3] = fast_ex2(fmaf(s[nt][3], SL2, -b_hi));
          ps_lo += s[nt][0] + s[nt][1];
          ps_hi += s[nt][2] + s[nt][3];
        }
      }
      l_lo = l_lo * sc_lo + ps_lo;
      l_hi = l_hi * sc_hi + ps_hi;
      if (c > 0) {
#pragma unroll
        for (int dt = 0; dt < 8; ++dt) {
          o[dt][0] *= sc_lo; o[dt][1] *= sc_lo; o[dt][2] *= sc_hi; o[dt][3] *= sc_hi;
        }
      }
      // ---- O += P V: 16-key steps, n-tiles 2 kk and 2 kk + 1 of S form the A fragment ----
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        if (kk < kn) {
          uint32_t pa[4];
          pa[0] = pack_f16x2(s[2 * kk][0], s[2 * kk][1]);
          pa[1] = pack_f16x2(s[2 * kk][2], s[2 * kk][3]);
          pa[2] = pack_f16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
          pa[3] = pack_f16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
          const int step = c * 8 + kk;  // 16-key step inside the sequence
          const uint32_t vbox = vs_u + (step >> 2) * VBOX_BYTES;
          const int chunk = (step & 3) * 2 + ((lane >> 3) & 1);
#pragma unroll
          for (int dp = 0; dp < 4; ++dp) {
            uint32_t b0, b1, b2, b3;
            ldsm_x4(vbox + swz((2 * dp + (lane >> 4)) * 8 + (lane & 7), chunk), b0, b1, b2, b3);
            mma_f16(o[2 * dp], pa, b0, b1);
            mma_f16(o[2 * dp + 1], pa, b2, b3);
          }
        }
      }
    }

    // ---- finalize ----
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float inv_lo = 1.0f / l_lo, inv_hi = 1.0f / l_hi;
    if (out_mode == 3) {
      // stage the 16 x 64 fp16 slice in the Q slot (Q is in registers), then whole 128-byte rows to global
#pragma unroll
      for (int dp = 0; dp < 4; ++dp)
        stsm_x4(qs_u + swz(lane & 15, 2 * dp + (lane >> 4)),
                pack_f16x2(o[2 * dp][0] * inv_lo, o[2 * dp][1] * inv_lo),
                pack_f16x2(o[2 * dp][2] * inv_hi, o[2 * dp][3] * inv_hi),
                pack_f16x2(o[2 * dp + 1][0] * inv_lo, o[2 * dp + 1][1] * inv_lo),
                pack_f16x2(o[2 * dp + 1][2] * inv_hi, o[2 * dp + 1][3] * inv_hi));
      __syncwarp();
      uint16_t* c16 = static_cast<uint16_t*>(ctx);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int idx = i * 32 + lane, r = idx >> 3, ch = idx & 7;
        if (sl * 16 + r < len) {
          const uint4 v = *reinterpret_cast<const uint4*>(qslot + swz(r, ch));
          *reinterpret_cast<uint4*>(c16 + (long long)(start + sl * 16 + r) * ldc + h * HD + ch * 8) = v;
        }
      }
    } else {
      const int row_lo = sl * 16 + g, row_hi = row_lo + 8;
      float* c32 = static_cast<float*>(ctx);
      const long long r_lo = (long long)(start + row_lo) * ldc, r_hi = (long long)(start + row_hi) * ldc;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) {
        const int col = h * HD + dt * 8 + 2 * t;
        float2 a = make_float2(o[dt][0] * inv_lo, o[dt][1] * inv_lo);
        float2 b = make_float2(o[dt][2] * inv_hi, o[dt][3] * inv_hi);
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
    __syncwarp();  // every lane is done with the Q slot (ldmatrix / staging reads) before the next slice's copies
  }
}

}  // namespace

// Which fp16 kernel takes a batch.  By default this one takes rows of 129 .. 208 tokens, where padding keys and
// queries to 64 costs the tile kernel of attention_f16.cu the most (ViT-B/16: 197 tokens, 256 x 256 scores there,
// 208 x 208 here).  Measured on an H100 SXM (700 W): 0.88x the tile kernel's time at 2,048 x 197 tokens x 12 heads,
// but 1.07x at 256 x 249 and 1.09x at 256 sentences of <= 32 tokens, which therefore stay on the tile kernel.
// MER_ATT_SHORT=1 sends every row of <= 249 tokens here, MER_ATT_SHORT=0 none.  Read at every launch, so that a
// test or a timing script can run both kernels in one process.
bool mer_attention_short_enabled(int max_seqlen) {
  if (max_seqlen <= 0 || max_seqlen > MAX_SEQ) return false;
  const char* e = getenv("MER_ATT_SHORT");
  if (e != nullptr && *e) return atoi(e) != 0;
  return max_seqlen > 128 && max_seqlen <= 208;
}

int mer_attention_short_launch(const void* qkv16, const void* vt16, long long vt_ld, void* ctx, const int* cu_seqlens,
                               int n_seq, long long tokens, int heads, int max_seqlen, int out_mode,
                               cudaStream_t stream) {
  MER_REQUIRE(qkv16 && vt16 && ctx && cu_seqlens, "mer_attention (short): null operand");
  MER_REQUIRE(out_mode >= 0 && out_mode <= 3, "mer_attention (short): out_mode %d", out_mode);
  MER_REQUIRE(vt_ld >= tokens && vt_ld % 8 == 0, "mer_attention (short): V^T pitch %lld must be a multiple of 8 >= tokens",
              vt_ld);
  MER_REQUIRE(max_seqlen > 0 && max_seqlen <= MAX_SEQ, "mer_attention (short): max_seqlen %d (1 .. %d)", max_seqlen,
              MAX_SEQ);
  MER_REQUIRE(heads > 0 && heads <= 65535 && n_seq <= 65535 && tokens < (1ll << 31),
              "mer_attention (short): bad grid (%d heads, %d seqs, %lld tokens)", heads, n_seq, tokens);
  if (n_seq <= 0 || tokens <= 0) return 0;
  static MerPerDevice attr_set;
  if (attr_set.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(attention_short_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        smem_bytes(KPOS_MAX)));
    MER_CUDA_CHECK(cudaFuncSetAttribute(attention_short_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                        cudaSharedmemCarveoutMaxShared));
    attr_set.mark();
  }
  const int kcap = (max_seqlen + 7 + 15) / 16 * 16;  // + up to 7 leading keys of the 8-token aligned start
  const double s_avg = (double)tokens / n_seq;  // exact for equal-length batches (ViT frames)
  const int prof = mer_prof_begin(MER_PROF_ATT_F16, 4.0 * s_avg * s_avg * HD * (double)n_seq * heads, stream);
  attention_short_kernel<<<dim3(heads, n_seq), THREADS, smem_bytes(kcap), stream>>>(
      static_cast<const uint16_t*>(qkv16), static_cast<const uint16_t*>(vt16), vt_ld, tokens, ctx, cu_seqlens, heads,
      kcap, out_mode);
  mer_prof_end(prof, stream);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  return 0;
}
