// gemm.cu — the one GEMM every encoder layer goes through.
//
//   out[b*out_bstride + out_row0 + m, n] =
//       fmt( act( sum_k A[b, m, k] * W[n, k] + bias[n] ) + res[b*res_bstride + res_row0 + m, n] )
//   act: none | erf-GELU | quick-GELU | ReLU (ReLU after the residual);  fmt: fp32 | tf32-rounded | bf16 hi|lo | fp16
//
// A is a (K, rows, batches) tensor described by a TMA map with ARBITRARY row / batch strides,
// which is how the strided HuBERT convolutions (time-major activations, overlapping windows),
// the HuBERT positional conv (block-diagonal windows, negative row offset = zero padding), the
// ViT / CLIP patch embeddings and the ResNet im2col operands run through the same kernel as the
// Linear layers (reference ops: HF ViT/CLIP/HuBERT/BERT nn.Linear + nn.Conv1d, torchvision Conv2d;
// see DESIGN.md kernel table).
// W is the nn.Linear weight as stored: [N, K] row-major == K-major B operand.
//
// Structure (persistent, warp-specialised, one CTA per SM, 128 x BLOCK_N output tiles):
//   warpgroup 0 (warp 0)  TMA producer: A/B tiles -> 128B-swizzled smem ring (mbarrier full/empty)
//   warpgroups 1, 2       consumers: rows [0, 64) / [64, 128) of the tile; wgmma.mma_async 64 x 128 x (32 bytes
//                         of K) per instruction (two per K step for BLOCK_N = 256), fp32 accumulators in
//                         registers; then the epilogue (bias / activation / residual / output format): outputs
//                         without residual or activation go through shared-memory slots and TMA stores (64-row
//                         sub-tiles); every other form is stored straight from the accumulator fragment
// The producer runs ahead across tile boundaries, so the next tile's operands stream in during the epilogue.
//
// Three arithmetic modes share the pipeline (128 bytes of K per smem row and stage in each):
//   MER_GEMM_F16    : IEEE fp16 operands (64 K elements per stage), wgmma f16.  Same 10-bit mantissa as
//                     tf32, twice the MMA rate, half the operand bytes: the ViT stack's default.
//   MER_GEMM_TF32   : fp32 operands (pre-rounded to tf32 by their producers), wgmma tf32, 128B swizzle.
//                     ~2.4e-4 relative error per GEMM: enough for the pre-LN ViT at 1e-3.
//   MER_GEMM_BF16X3 : every operand stored as bf16 (hi, lo) pairs, x = hi + lo to 2^-17, in 128-byte
//                     groups [32 hi | 32 lo] so that tiles move exactly like TF32 tiles; three
//                     bf16 MMAs per 16-wide K step (hi*hi + lo*hi + hi*lo), fp32 accumulate.
//                     ~2e-5 relative error per GEMM: what the post-LN HuBERT/BERT stacks need to stay
//                     inside 1e-3 after 12 layers (measured: single-pass TF32 reaches 1.0e-3 after 4).
#include <stdlib.h>

#include "mer_common.cuh"
#include "mer_kernels.h"

namespace {

using namespace mer;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 32;  // K elements per stage in TF32 / BF16X3 mode (128 B of tf32 / 64 B of bf16 per part)
constexpr int CONSUMERS = 2;  // consumer warpgroups, 64 tile rows each
constexpr int NUM_THREADS = 128 * (1 + CONSUMERS);

template <int BLOCK_N, int MODE>
struct GemmCfg {
  static constexpr bool kSplit = MODE == MER_GEMM_BF16X3;
  static constexpr bool kF16 = MODE == MER_GEMM_F16;
  static constexpr int kBlockK = kF16 ? 64 : BLOCK_K;  // K elements per stage
  static constexpr int kRowBytes = 128;                 // bytes of K per smem row = swizzle span
  static constexpr int kKind = kSplit ? 1 : (kF16 ? 0 : 2);  // wgmma operand type: f16 / bf16 / tf32
  static constexpr int kABytes = BLOCK_M * kRowBytes;
  static constexpr int kBBytes = BLOCK_N * kRowBytes;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = BLOCK_N == 256 ? 4 : 6;  // 192 KB of operands either way (227 KB usable)
  static constexpr int kSlotsBytes = 2 * 2 * 64 * 128;     // TMA epilogue: 2 slot pairs of 2 x 8 KB
  static constexpr int kBarBytes = 256;
  static constexpr int smem_bytes(bool tma) { return kStages * kStageBytes + (tma ? kSlotsBytes : 0) + kBarBytes + 1024; }
  static_assert(smem_bytes(true) <= 227 * 1024, "shared memory budget");
};

// internal epilogue flag (set by mer_gemm_launch when MER_GELU_PACKED=1): erf-GELU on value pairs through the
// paired polynomial (GELU kind 5; fp16 and split-bf16 outputs, no residual).  Off by default.
constexpr int EPI_GELU_PACKED = 1 << 16;

// BLOOM's bloom_gelu_forward, 0.5 x (1 + tanh(u)) with u = 0.79788456 x (1 + 0.044715 x^2) (u formed in HF's order).
// As x sigmoid(2u): with t = exp(-2|u|) and r = t / (1 + t) in [0, 1/2], the result is x - x r for x >= 0 and x r
// below.  Only the small term x r carries the ex2 / rcp approximation error, so |error| stays within an ulp of the
// result (<= 1e-6 on [-20, 20] against torch's fp32 tanh form); tanh.approx.f32 would not.
__device__ __forceinline__ float gelu_tanh(float x) {
  const float u = (0.79788456f * x) * (1.0f + (0.044715f * x) * x);
  float t, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(-2.8853900817779268f * fabsf(u)));  // exp(-2|u|)
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + t));
  r *= t;
  return x >= 0.f ? fmaf(-x, r, x) : x * r;
}

template <int GELU>
__device__ __forceinline__ float epi_act(float v) {
  if (GELU == 1) return gelu_erf_fast(v);
  if (GELU == 2) return gelu_erf(v);
  if (GELU == 3) return quick_gelu_fast(v);
  if (GELU == 6) return gelu_tanh(v);
  return v;  // GELU == 4 (ReLU) is applied after the residual add
}
// two adjacent values at once (GELU == 5: the paired polynomial; otherwise the scalar form twice)
template <int GELU>
__device__ __forceinline__ void epi_act2(float a, float b, float& ga, float& gb) {
  if (GELU == 5) {
    gelu_erf_fast2(a, b, ga, gb);
  } else {
    ga = epi_act<GELU>(a);
    gb = epi_act<GELU>(b);
  }
}

// Epilogue of one consumer warpgroup for its 64 x BLOCK_N share of a tile, straight from the wgmma accumulator
// fragment: acc[h][4 j + 2 i + c] holds row 16 warp + g + 8 i, column 128 h + 8 j + 2 t + c (g = lane / 4,
// t = lane % 4).  Each thread handles column pairs; one store instruction covers 8 rows x 32 contiguous bytes.
// GELU: 0 none, 1 polynomial erf, 2 libdevice erff, 3 quick-GELU, 4 ReLU (after the residual), 5 paired erf,
// 6 tanh-GELU (BLOOM).
// OUT: 0 fp32, 1 TF32-rounded fp32, 2 bf16 (hi|lo), 3 fp16.  RES: add the residual after the activation.
// The transposed side output (V^T of the QKV GEMM) exists for GELU == 0 without residual: columns >= vt_col0 go
// to vt[n - vt_col0, out_row] INSTEAD of out.
template <int NH, int GELU, int OUT, bool RES>
__device__ __forceinline__ void epi_tile(float (&acc)[NH][64], const MerGemmEpilogue& ep, int n_base, int m_base,
                                         int rows_per_batch, long long out_row_b, long long res_row_b, int wg_row0) {
  constexpr bool kVt = GELU == 0 && !RES;
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = m_base + wg_row0 + 16 * w + g + 8 * i;  // row inside the batch entry
    if (m >= rows_per_batch) continue;
    const long long orow = out_row_b + m;
    const float* rrow = RES ? ep.res + (res_row_b + m) * (long long)ep.ld_res : nullptr;
#pragma unroll
    for (int hh = 0; hh < NH; ++hh) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int n = n_base + 128 * hh + 8 * j + 2 * t;
        float v0 = acc[hh][4 * j + 2 * i], v1 = acc[hh][4 * j + 2 * i + 1];
        if (ep.bias) {
          const float2 q = __ldg(reinterpret_cast<const float2*>(ep.bias + n));
          v0 += q.x;
          v1 += q.y;
        }
        if (kVt && ep.vt != nullptr && n >= ep.vt_col0) {
          const long long vo = (long long)(n - ep.vt_col0) * ep.vt_ld + orow;
          if (OUT == 3) {
            uint16_t* vt16 = reinterpret_cast<uint16_t*>(ep.vt) + vo;
            const uint32_t p = pack_f16x2(v0, v1);
            vt16[0] = (uint16_t)(p & 0xffffu);
            vt16[ep.vt_ld] = (uint16_t)(p >> 16);
          } else {
            if (OUT == 1) {
              v0 = round_tf32(v0);
              v1 = round_tf32(v1);
            }
            ep.vt[vo] = v0;
            ep.vt[vo + ep.vt_ld] = v1;
          }
          continue;
        }
        epi_act2<GELU>(v0, v1, v0, v1);
        if (RES) {
          const float2 r = __ldg(reinterpret_cast<const float2*>(rrow + n));
          v0 += r.x;
          v1 += r.y;
        }
        if (GELU == 4) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        if (OUT == 3) {
          *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(ep.out) + orow * ep.ld_out + n) = pack_f16x2(v0, v1);
        } else if (OUT == 2) {
          store_split2(ep.out + orow * ep.ld_out, n, v0, v1);
        } else {
          if (OUT == 1) {
            v0 = round_tf32(v0);
            v1 = round_tf32(v1);
          }
          *reinterpret_cast<float2*>(ep.out + orow * ep.ld_out + n) = make_float2(v0, v1);
        }
      }
    }
  }
}

// ---- TMA epilogue (outputs without residual or activation: the QKV form) ----
// Output slots: 64 rows x 128 bytes (32 fp32 / 64 fp16 columns) in the 128B-swizzled layout of one TMA box, so a slot
// is one cp.async.bulk.tensor store.  Slots come in pairs, one per consumer warpgroup; a warpgroup's u-th sub-tile
// (u counts on across tiles) uses pair u % kSlotPairs.  The warpgroup waits only until a slot has been read out by its
// previous store, never for the global write, so a tile's output traffic runs under the next tile's MMAs.
constexpr int kSlotBytes = 64 * 128;
constexpr int kSlotPairs = 2;

__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the bulk stores committed before the last N groups have finished reading shared memory
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// named barrier over the 128 threads of consumer warpgroup wg (1 | 2); id 0 is __syncthreads
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg) : "memory"); }

// epi_tile<NH, 0, OUT, false>'s arithmetic on one pair (bias, then the tf32 rounding of OUT == 1), in its order
template <int OUT>
__device__ __forceinline__ void epi_bias_round(float& v0, float& v1, const float* bias, int n) {
  if (bias) {
    const float2 q = __ldg(reinterpret_cast<const float2*>(bias + n));
    v0 += q.x;
    v1 += q.y;
  }
  if (OUT == 1) {
    v0 = round_tf32(v0);
    v1 = round_tf32(v1);
  }
}

// TMA epilogue of one consumer warpgroup (OUT: 0 fp32, 1 TF32-rounded fp32, 3 fp16; no activation, no residual): the
// same fragment and values as epi_tile<NH, 0, OUT, false>, but each 64 x (32 fp32 | 64 fp16) sub-tile is written into
// a slot and stored by one thread with TMA, which clips rows past rows_per_batch.  Sub-tiles at or past vt_col0 (a
// multiple of the sub-tile width) keep epi_tile's V^T stores and use no slot.  slots: this warpgroup's slot of pair 0;
// q: slot uses so far.
template <int NH, int OUT>
__device__ __forceinline__ void epi_tile_tma(float (&acc)[NH][64], const MerGemmEpilogue& ep, const CUtensorMap* tmap_out,
                                             uint8_t* slots, uint32_t& q, int n_base, int m_base, int b,
                                             int rows_per_batch, long long out_row_b, int wg_row0, int wg) {
  static_assert(OUT == 0 || OUT == 1 || OUT == 3, "fp32, tf32 or fp16 output");
  constexpr int kEl = OUT == 3 ? 2 : 4;
  constexpr int kCols = 128 / kEl;  // columns per slot
  constexpr int kJ = kCols / 8;     // 8-column fragment groups per slot
  constexpr int kSub = NH * 128 / kCols;
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int g = lane >> 2, t = lane & 3;
  const bool leader = (threadIdx.x & 127) == 0;
#pragma unroll
  for (int s = 0; s < kSub; ++s) {
    const int hh = s * kCols / 128, j0 = (s * kCols % 128) / 8;
    const int n0 = n_base + s * kCols;
    if (ep.vt != nullptr && n0 >= ep.vt_col0) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int m = m_base + wg_row0 + 16 * w + g + 8 * i;
        if (m >= rows_per_batch) continue;
        const long long orow = out_row_b + m;
#pragma unroll
        for (int jj = 0; jj < kJ; ++jj) {
          const int n = n0 + 8 * jj + 2 * t;
          float v0 = acc[hh][4 * (j0 + jj) + 2 * i], v1 = acc[hh][4 * (j0 + jj) + 2 * i + 1];
          epi_bias_round<OUT>(v0, v1, ep.bias, n);
          const long long vo = (long long)(n - ep.vt_col0) * ep.vt_ld + orow;
          if (OUT == 3) {
            uint16_t* vt16 = reinterpret_cast<uint16_t*>(ep.vt) + vo;
            const uint32_t p = pack_f16x2(v0, v1);
            vt16[0] = (uint16_t)(p & 0xffffu);
            vt16[ep.vt_ld] = (uint16_t)(p >> 16);
          } else {
            ep.vt[vo] = v0;
            ep.vt[vo + ep.vt_ld] = v1;
          }
        }
      }
      continue;
    }
    uint8_t* slot = slots + (q % kSlotPairs) * 2 * kSlotBytes;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 16 * w + g + 8 * i;  // slot row; r % 8 == g
#pragma unroll
      for (int jj = 0; jj < kJ; ++jj) {
        float v0 = acc[hh][4 * (j0 + jj) + 2 * i], v1 = acc[hh][4 * (j0 + jj) + 2 * i + 1];
        epi_bias_round<OUT>(v0, v1, ep.bias, n0 + 8 * jj + 2 * t);
        // byte (8 jj + 2 t) * kEl of the row, 16-byte chunks XOR-swizzled by r % 8
        const int byte = (8 * jj + 2 * t) * kEl;
        uint8_t* at = slot + r * 128 + ((((byte >> 4) ^ g) << 4) | (byte & 15));
        if (OUT == 3) *reinterpret_cast<uint32_t*>(at) = pack_f16x2(v0, v1);
        else *reinterpret_cast<float2*>(at) = make_float2(v0, v1);
      }
    }
    fence_proxy_async();
    // before the barrier: the slot of the NEXT use has been read out by its previous store
    if (leader) bulk_wait_read<kSlotPairs - 2>();
    wg_sync(wg);
    if (leader) {
      tma_store_3d(tmap_out, slot, n0, m_base + wg_row0, b);
      bulk_commit();
    }
    ++q;
  }
}

// TMA: the TMA epilogue (epi_tile_tma, for a descriptor without residual or activation) instead of epi_tile.  Two
// kernels rather than a run-time switch, so that the register epilogue keeps its own code and register allocation.
template <int BLOCK_N, int MODE, bool TMA>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a,
            const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ CUtensorMap tmap_out,
            const MerGemmEpilogue ep,
            int rows_per_batch, int batches, int N, int K, int K_inner, int P, int a_row0, int a_col_group) {
  using Cfg = GemmCfg<BLOCK_N, MODE>;
  static_assert(Cfg::kSlotsBytes == 2 * kSlotPairs * kSlotBytes, "epilogue slot budget");
  constexpr int NH = BLOCK_N / 128;  // 64 x 128 accumulator blocks per consumer thread
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by OFFSET (not through an integer round trip) so the compiler keeps the
  // shared address space of everything derived from it
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kABytes;
  uint8_t* slots = smem + Cfg::kStages * Cfg::kStageBytes;  // TMA: [pair][warpgroup] x kSlotBytes
  uint64_t* bars = reinterpret_cast<uint64_t*>(slots + (TMA ? Cfg::kSlotsBytes : 0));
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int m_tiles = (rows_per_batch + BLOCK_M - 1) / BLOCK_M;
  const int n_tiles = N / BLOCK_N;
  const int num_kb = K / Cfg::kBlockK;
  const int num_tiles = batches * m_tiles * n_tiles;  // work item t: column block t % n_tiles, row tile t / n_tiles

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (TMA) tma_prefetch_desc(&tmap_out);
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full_bar[i], 1);                // the producer's expect-tx arrival
      mbar_init(&empty_bar[i], 4 * CONSUMERS);   // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp != 0) return;
    // The whole warp runs the loop (so addresses and coordinates stay in uniform registers); one
    // elected lane issues the copies.  No division inside the K loop.
    int stage = 0;
    uint32_t phase = 0;
    constexpr int kEl = Cfg::kSplit ? 2 : 1;  // tensor-map elements per operand value
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const int n_blk = t % n_tiles;
      const int mb = t / n_tiles;
      const int b = mb / m_tiles;
      const int mt = mb % m_tiles;
      int c0 = 0, tap_phase = 0, tap_row = 0;  // K offset inside the tap; tap % P; tap / P
      // block-diagonal (grouped conv) mode: this column block's window of A columns
      const int c_win = a_col_group > 0 ? ((n_blk * BLOCK_N) / a_col_group) * a_col_group : 0;
      const int row_base = mt * BLOCK_M + a_row0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait_nocall(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_4d(smem_a + stage * Cfg::kABytes, &tmap_a, &full_bar[stage], (c_win + c0) * kEl, tap_phase,
                      row_base + tap_row, b);
          tma_load_2d(smem_b + stage * Cfg::kBBytes, &tmap_b, &full_bar[stage], kb * Cfg::kBlockK * kEl,
                      n_blk * BLOCK_N);
        }
        __syncwarp();
        c0 += Cfg::kBlockK;
        if (c0 == K_inner) {
          c0 = 0;
          if (++tap_phase == P) {
            tap_phase = 0;
            ++tap_row;
          }
        }
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int wg_row0 = (wg - 1) * 64;  // this warpgroup's rows of the tile
  const uint64_t desc_a0 = wgmma_desc_sw128(smem_u32(smem_a + wg_row0 * Cfg::kRowBytes));
  const uint64_t desc_b0 = wgmma_desc_sw128(smem_u32(smem_b));
  const int gelu_kind = (ep.flags & MER_EPI_GELU_TANH) ? 6 : (ep.flags & MER_EPI_RELU) ? 4
                        : (ep.flags & MER_EPI_QUICK_GELU) ? 3
                        : (ep.flags & MER_EPI_GELU)
                            ? ((ep.flags & MER_EPI_GELU_LIBM) ? 2 : ((ep.flags & EPI_GELU_PACKED) ? 5 : 1)) : 0;
  const int out_kind = (ep.flags & MER_EPI_OUT_F16) ? 3 : (ep.flags & MER_EPI_SPLIT_BF16) ? 2 :
                       ((ep.flags & MER_EPI_ROUND_TF32) ? 1 : 0);
  const int kind = gelu_kind * 4 + out_kind;
  int stage = 0;
  uint32_t phase = 0;
  uint32_t slot_uses = 0;  // TMA: this warpgroup's slot uses so far
  float acc[NH][64];
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int n_blk = t % n_tiles;
    const int mb = t / n_tiles;
    const int b = mb / m_tiles;
    const int mt = mb % m_tiles;
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait_nocall(&full_bar[stage], phase);
      // descriptors: start address field counts 16-byte units; a stage is kABytes / kBBytes further
      const uint64_t da = desc_a0 + (uint64_t)(stage * (Cfg::kABytes >> 4));
      const uint64_t db = desc_b0 + (uint64_t)(stage * (Cfg::kBBytes >> 4));
      constexpr uint64_t kHalfB = (128 * Cfg::kRowBytes) >> 4;  // B rows [128, 256) of the stage
      wgmma_fence();
      // advance the start address by 32-byte K steps inside the 128B swizzle row (>>4 => +2)
#pragma unroll
      for (int k = 0; k < (Cfg::kSplit ? 2 : 4); ++k) {
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) {
          const uint64_t dbh = db + hh * kHalfB;
          if (!Cfg::kSplit) {
            wgmma_m64n128<Cfg::kKind>(acc[hh], da + 2 * k, dbh + 2 * k, (kb | k) != 0);
          } else {  // 2 x 16 bf16; hi at bytes [0,64), lo at [64,128) of the row
            wgmma_m64n128<1>(acc[hh], da + 2 * k, dbh + 2 * k, (kb | k) != 0);  // hi * hi
            wgmma_m64n128<1>(acc[hh], da + 4 + 2 * k, dbh + 2 * k, 1);          // lo * hi
            wgmma_m64n128<1>(acc[hh], da + 2 * k, dbh + 4 + 2 * k, 1);          // hi * lo
          }
        }
      }
      wgmma_commit();
      // the previous stage's MMAs have retired once at most this stage's group is in flight: free its slot
      wgmma_wait<1>();
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == Cfg::kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int hh = 0; hh < NH; ++hh)
#pragma unroll
      for (int r = 0; r < 64; ++r) wgmma_fence_operand(acc[hh][r]);
    if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

    const int n_base = n_blk * BLOCK_N;
    const int m_base = mt * BLOCK_M;
    const long long out_row_b = (long long)b * ep.out_bstride + ep.out_row0;
    const long long res_row_b = (long long)b * ep.res_bstride + ep.res_row0;
    if constexpr (TMA) {  // the host sends only fp32 / tf32 / fp16 outputs without residual or activation here
      if (out_kind == 3)
        epi_tile_tma<NH, 3>(acc, ep, &tmap_out, slots + (wg - 1) * kSlotBytes, slot_uses, n_base, m_base, b,
                            rows_per_batch, out_row_b, wg_row0, wg);
      else if (out_kind == 1)
        epi_tile_tma<NH, 1>(acc, ep, &tmap_out, slots + (wg - 1) * kSlotBytes, slot_uses, n_base, m_base, b,
                            rows_per_batch, out_row_b, wg_row0, wg);
      else
        epi_tile_tma<NH, 0>(acc, ep, &tmap_out, slots + (wg - 1) * kSlotBytes, slot_uses, n_base, m_base, b,
                            rows_per_batch, out_row_b, wg_row0, wg);
    } else {
#define MER_EPI(G, O, R) epi_tile<NH, G, O, R>(acc, ep, n_base, m_base, rows_per_batch, out_row_b, res_row_b, wg_row0)
    if (ep.res != nullptr) {  // uniform across the kernel; each variant is straight-line code
      if (gelu_kind == 4) MER_EPI(4, 0, true);        // relu(acc + bias + res)
      else if (gelu_kind != 0) MER_EPI(1, 0, true);   // res + GELU(acc + bias), erf form
      else if (out_kind == 1) MER_EPI(0, 1, true);
      else MER_EPI(0, 0, true);
    } else {
      switch (kind) {
        case 0: MER_EPI(0, 0, false); break;
        case 1: MER_EPI(0, 1, false); break;
        case 2: MER_EPI(0, 2, false); break;
        case 3: MER_EPI(0, 3, false); break;
        case 4: MER_EPI(1, 0, false); break;
        case 5: MER_EPI(1, 1, false); break;
        case 6: MER_EPI(1, 2, false); break;
        case 7: MER_EPI(1, 3, false); break;
        case 8: MER_EPI(2, 0, false); break;
        case 9: MER_EPI(2, 1, false); break;
        case 10: MER_EPI(2, 2, false); break;
        case 11: MER_EPI(2, 3, false); break;
        case 13: MER_EPI(3, 1, false); break;   // quick-GELU: the operand
        case 15: MER_EPI(3, 3, false); break;   // formats FC1 can feed
        case 16: MER_EPI(4, 0, false); break;   // relu(acc + bias)
        case 19: MER_EPI(4, 3, false); break;   // the same as the fp16 operand of the next GEMM (OPT fc1)
        case 24: MER_EPI(6, 0, false); break;   // tanh-GELU (BLOOM dense_h_to_4h)
        case 27: MER_EPI(6, 3, false); break;
        case 22: MER_EPI(5, 2, false); break;   // paired erf-GELU (opt-in)
        case 23: MER_EPI(5, 3, false); break;
        default: MER_EPI(3, 0, false); break;
      }
    }
#undef MER_EPI
    }
  }
  if (TMA && (threadIdx.x & 127) == 0) bulk_wait_all();  // the last stores have landed before the CTA retires
}

// launches per kernel instantiation (tests assert that the variant a configuration is benchmarked on is the one a
// parity test exercised): index = mode | (BLOCK_N == 256) << 2
long long g_variant_launches[8] = {};
// launches per epilogue: [0] register, [1] TMA
long long g_epilogue_launches[2] = {};

// Whether a launch takes the TMA epilogue: an fp32, tf32 or fp16 output without residual or activation (the QKV form;
// measured on an H100, the residual and activation forms ran no faster through the slots, see DESIGN §7), the out base
// (at out_row0) 16-byte aligned, its row and batch pitches multiples of 16 bytes and no narrower than N, and V^T (if
// any) starting at a sub-tile boundary (32 fp32 / 64 fp16 columns).  MER_GEMM_EPI_TMA=0, read at every launch so that
// both epilogues can be compared in one process, forces the register epilogue.
bool use_tma_epilogue(const MerGemmDesc* g) {
  const MerGemmEpilogue& ep = g->ep;
  const char* e = getenv("MER_GEMM_EPI_TMA");
  if ((e && *e && atoi(e) == 0) || ep.res ||
      (ep.flags & (MER_EPI_SPLIT_BF16 | MER_EPI_GELU | MER_EPI_QUICK_GELU | MER_EPI_RELU | MER_EPI_GELU_TANH)))
    return false;
  const long long el = (ep.flags & MER_EPI_OUT_F16) ? 2 : 4;
  if ((reinterpret_cast<uintptr_t>(ep.out) + ep.out_row0 * ep.ld_out * el) % 16 || ep.ld_out * el % 16 ||
      ep.ld_out < g->N || (g->batches > 1 && ep.out_bstride * ep.ld_out * el % 16))
    return false;
  return ep.vt == nullptr || ep.vt_col0 % (128 / el) == 0;
}

template <int BLOCK_N, int MODE>
int launch_gemm(const MerGemmDesc* g, cudaStream_t stream) {
  using Cfg = GemmCfg<BLOCK_N, MODE>;
  ++g_variant_launches[(MODE & 3) | (BLOCK_N == 256 ? 4 : 0)];
  CUtensorMap ta, tb, tout;
  memset(&tout, 0, sizeof(tout));
  const CUtensorMapDataType dt = Cfg::kSplit ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                 : Cfg::kF16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                             : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;
  const uint64_t mult = Cfg::kSplit ? 2 : 1;  // bf16 elements per 4-byte operand slot
  const uint64_t sbytes = Cfg::kF16 ? 2 : 4;  // bytes per stride unit (fp16 element / 4-byte slot)
  {
    // strides are given in 4-byte operand slots in both modes (a split row of K (hi|lo) pairs
    // occupies exactly the bytes of K fp32 values)
    const uint64_t dims[4] = {(uint64_t)(g->a_cols > 0 ? g->a_cols : g->K_inner) * mult, (uint64_t)g->P,
                              (uint64_t)g->a_rows_dim, (uint64_t)g->batches};
    const uint64_t strides[3] = {(uint64_t)g->a_phase_stride * sbytes,
                                 (uint64_t)g->a_row_stride * sbytes,
                                 (uint64_t)g->a_batch_stride * sbytes};
    const uint32_t box[4] = {(uint32_t)(Cfg::kBlockK * mult), 1, BLOCK_M, 1};
    if (int rc = mer_make_tmap(&ta, dt, 4, g->A, dims, strides, box, sw)) return rc;
  }
  {
    const int K = g->K_inner * g->taps;
    const uint64_t dims[2] = {(uint64_t)K * mult, (uint64_t)g->N};
    const uint64_t strides[1] = {(uint64_t)K * sbytes};
    const uint32_t box[2] = {(uint32_t)(Cfg::kBlockK * mult), BLOCK_N};
    if (int rc = mer_make_tmap(&tb, dt, 2, g->W, dims, strides, box, sw)) return rc;
  }
  // TMA epilogue map: (columns, rows_per_batch, batches) over the output from out_row0; the row dimension is exactly
  // rows_per_batch, so TMA clips the last row tile of every batch entry
  const bool tma = use_tma_epilogue(g);
  ++g_epilogue_launches[tma ? 1 : 0];
  if (tma) {
    const bool f16 = (g->ep.flags & MER_EPI_OUT_F16) != 0;
    const uint64_t el = f16 ? 2 : 4, ld = (uint64_t)g->ep.ld_out * el;
    const uint64_t dims[3] = {(uint64_t)g->N, (uint64_t)g->rows_per_batch, (uint64_t)g->batches};
    const uint64_t strides[2] = {ld, g->batches > 1 ? (uint64_t)g->ep.out_bstride * ld : (uint64_t)g->rows_per_batch * ld};
    const uint32_t box[3] = {(uint32_t)(128 / el), 64, 1};
    if (int rc = mer_make_tmap(&tout, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3,
                               reinterpret_cast<const char*>(g->ep.out) + g->ep.out_row0 * ld, dims, strides, box, sw))
      return rc;
  }
  static MerPerDevice attr_set;
  if (attr_set.needs_setup()) {
    MER_CUDA_CHECK(cudaFuncSetAttribute(gemm_kernel<BLOCK_N, MODE, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        Cfg::smem_bytes(false)));
    MER_CUDA_CHECK(cudaFuncSetAttribute(gemm_kernel<BLOCK_N, MODE, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        Cfg::smem_bytes(true)));
    attr_set.mark();
  }
  const int m_tiles = (g->rows_per_batch + BLOCK_M - 1) / BLOCK_M;
  const long long tiles = (long long)g->batches * m_tiles * (g->N / BLOCK_N);
  MER_REQUIRE(tiles < (1ll << 31), "mer_gemm: %lld tiles", tiles);
  int grid = mer_num_sms();
  if (tiles < grid) grid = (int)tiles;
  // profile class: the GEMM mode; fp16 problems of fewer than 2^17 rows (the HuBERT / BERT layers) are kept apart
  // as class 3 so that the dominant kernel's roofline is not an average over launches of very different sizes
  const int klass = (MODE == MER_GEMM_F16 && (long long)g->rows_per_batch * g->batches < (1ll << 17)) ? MER_PROF_F16_SMALL
                                                                                                        : MODE;
  const int prof = mer_prof_begin(klass, 2.0 * (double)g->rows_per_batch * g->batches * g->N *
                                             (double)(g->K_inner * g->taps), stream);
  MerGemmEpilogue ep = g->ep;
  {
    const bool plain_gelu = (ep.flags & MER_EPI_GELU) && !(ep.flags & MER_EPI_GELU_LIBM) && !ep.res;
    if (plain_gelu && (ep.flags & (MER_EPI_OUT_F16 | MER_EPI_SPLIT_BF16))) {
      // FC1 launches only; read at every such launch so that tests can run both forms in one process
      const char* e = getenv("MER_GELU_PACKED");
      if (e && atoi(e) == 1) ep.flags |= EPI_GELU_PACKED;
    }
  }
  (tma ? gemm_kernel<BLOCK_N, MODE, true> : gemm_kernel<BLOCK_N, MODE, false>)<<<grid, NUM_THREADS,
                                                                                 Cfg::smem_bytes(tma), stream>>>(
      ta, tb, tout, ep, g->rows_per_batch, g->batches, g->N, g->K_inner * g->taps, g->K_inner, g->P, g->a_row0,
      g->a_col_group);
  MER_CUDA_CHECK(cudaGetLastError());
  mer_count_launches(1);
  mer_prof_end(prof, stream);
  return 0;
}

}  // namespace

extern "C" long long mer_gemm_variant_launches(int block_n, int mode, int cluster, int twosm) {
  if ((block_n != 128 && block_n != 256) || mode < 0 || mode > 2 || cluster < 1 || cluster > 2) return -1;
  if (cluster != 1 || twosm) return 0;  // sm_90 build: single-CTA tiles only
  return g_variant_launches[(mode & 3) | (block_n == 256 ? 4 : 0)];
}

extern "C" long long mer_gemm_epilogue_launches(int tma) {
  if (tma != 0 && tma != 1) return -1;
  return g_epilogue_launches[tma];
}

int mer_gemm_launch(const MerGemmDesc* g, cudaStream_t stream) {
  MER_REQUIRE(g && g->A && g->W && g->ep.out, "mer_gemm: null operand");
  MER_REQUIRE(g->mode == MER_GEMM_TF32 || g->mode == MER_GEMM_BF16X3 || g->mode == MER_GEMM_F16,
              "mer_gemm: unknown mode %d", g->mode);
  const int kstep = g->mode == MER_GEMM_F16 ? 64 : BLOCK_K;
  const int salign = g->mode == MER_GEMM_F16 ? 8 : 4;  // stride units per 16 bytes

  MER_REQUIRE(g->K_inner > 0 && g->K_inner % kstep == 0 && g->taps > 0 && g->P > 0,
              "mer_gemm: K_inner=%d must be a positive multiple of %d (taps=%d P=%d)",
              g->K_inner, kstep, g->taps, g->P);
  MER_REQUIRE(g->a_rows_dim >= g->rows_per_batch, "mer_gemm: a_rows_dim < rows_per_batch");
  MER_REQUIRE(g->N > 0 && g->N % 128 == 0, "mer_gemm: N=%d must be a multiple of 128", g->N);
  MER_REQUIRE(g->rows_per_batch > 0 && g->batches > 0, "mer_gemm: empty problem");
  MER_REQUIRE(g->a_row_stride % salign == 0 && g->a_batch_stride % salign == 0 &&
                  g->a_phase_stride % salign == 0,
              "mer_gemm: A strides must be multiples of 16 bytes");
  MER_REQUIRE(!((g->ep.flags & MER_EPI_OUT_F16) &&
                ((g->ep.flags & (MER_EPI_SPLIT_BF16 | MER_EPI_ROUND_TF32)) || g->ep.res)),
              "mer_gemm: an fp16 output excludes the other output formats and a residual");
  MER_REQUIRE(g->ep.ld_out % 4 == 0 && (g->ep.res == nullptr || g->ep.ld_res % 4 == 0),
              "mer_gemm: out/res leading dims must be multiples of 4 floats");
  MER_REQUIRE(!((g->ep.flags & MER_EPI_SPLIT_BF16) && (g->ep.res || g->ep.vt)),
              "mer_gemm: a bf16-split output cannot be combined with a residual or the transposed side output");
  MER_REQUIRE(!(g->ep.res && g->ep.vt), "mer_gemm: a residual cannot be combined with the transposed side output");
  MER_REQUIRE(!(g->ep.res && (g->ep.flags & MER_EPI_GELU) &&
                (g->ep.flags & (MER_EPI_ROUND_TF32 | MER_EPI_GELU_LIBM))),
              "mer_gemm: residual + GELU is available with the polynomial GELU and a plain fp32 output");
  MER_REQUIRE(!((g->ep.flags & MER_EPI_QUICK_GELU) &&
                ((g->ep.flags & (MER_EPI_GELU | MER_EPI_SPLIT_BF16)) || g->ep.res || g->ep.vt)),
              "mer_gemm: quick-GELU comes alone (fp32, tf32 or fp16 output; no residual / split / V^T)");
  MER_REQUIRE(!((g->ep.flags & MER_EPI_RELU) &&
                ((g->ep.flags & (MER_EPI_GELU | MER_EPI_QUICK_GELU | MER_EPI_SPLIT_BF16 | MER_EPI_ROUND_TF32)) ||
                 g->ep.vt)),
              "mer_gemm: ReLU goes with a plain fp32 output (optionally + residual) or an fp16 output");
  MER_REQUIRE(!((g->ep.flags & MER_EPI_GELU_TANH) &&
                ((g->ep.flags & (MER_EPI_GELU | MER_EPI_GELU_LIBM | MER_EPI_QUICK_GELU | MER_EPI_RELU |
                                 MER_EPI_SPLIT_BF16 | MER_EPI_ROUND_TF32)) || g->ep.res || g->ep.vt)),
              "mer_gemm: tanh-GELU comes alone (fp32 or fp16 output, optional bias; no residual / split / tf32 / V^T)");
  MER_REQUIRE(g->a_col_group == 0 || g->force_block_n == 128 || g->force_block_n == 256,
              "mer_gemm: a_col_group needs force_block_n (the weights are built for one block width)");
  MER_REQUIRE(!(g->ep.vt && (g->ep.flags & MER_EPI_GELU)), "mer_gemm: GELU + transposed side output is not supported");
  // the epilogue routes whole column pairs (n, n + 1), n even, to vt or out and writes vt row n - vt_col0
  MER_REQUIRE(g->ep.vt == nullptr || (g->ep.vt_col0 >= 0 && g->ep.vt_col0 < g->N && g->ep.vt_col0 % 2 == 0),
              "mer_gemm: vt_col0=%d must be even and in [0, N=%d)", g->ep.vt_col0, g->N);
  // flags the kernel would otherwise ignore or resolve silently
  MER_REQUIRE(!((g->ep.flags & MER_EPI_GELU_LIBM) && !(g->ep.flags & MER_EPI_GELU)),
              "mer_gemm: MER_EPI_GELU_LIBM selects the erf form of MER_EPI_GELU and needs it");
  MER_REQUIRE(!((g->ep.flags & MER_EPI_ROUND_TF32) && (g->ep.flags & MER_EPI_SPLIT_BF16)),
              "mer_gemm: a tf32-rounded output excludes the bf16-split output");
  // the epilogue loads bias / res as float2 and stores out as float2 (fp32) or as an fp16 pair (uint32)
  const uintptr_t out_align = (g->ep.flags & MER_EPI_OUT_F16) ? 4 : 8;
  MER_REQUIRE(reinterpret_cast<uintptr_t>(g->ep.out) % out_align == 0 &&
                  reinterpret_cast<uintptr_t>(g->ep.res) % 8 == 0 && reinterpret_cast<uintptr_t>(g->ep.bias) % 8 == 0,
              "mer_gemm: out must be %d-byte aligned, res and bias 8-byte aligned (out %p res %p bias %p)",
              (int)out_align, (const void*)g->ep.out, (const void*)g->ep.res, (const void*)g->ep.bias);
  const int m_tiles = (g->rows_per_batch + BLOCK_M - 1) / BLOCK_M;
  const long long tiles256 = (g->N % 256 == 0) ? (long long)g->batches * m_tiles * (g->N / 256) : 0;
  // 128 x 256 tiles whenever they fill the machine; 128 x 128 for small problems / N % 256 != 0
  const bool wide = (tiles256 >= mer_num_sms() && g->force_block_n != 128) ||
                    (g->force_block_n == 256 && tiles256 > 0);
  if (g->mode == MER_GEMM_F16)
    return wide ? launch_gemm<256, MER_GEMM_F16>(g, stream) : launch_gemm<128, MER_GEMM_F16>(g, stream);
  if (g->mode == MER_GEMM_BF16X3)
    return wide ? launch_gemm<256, MER_GEMM_BF16X3>(g, stream) : launch_gemm<128, MER_GEMM_BF16X3>(g, stream);
  return wide ? launch_gemm<256, MER_GEMM_TF32>(g, stream) : launch_gemm<128, MER_GEMM_TF32>(g, stream);
}
