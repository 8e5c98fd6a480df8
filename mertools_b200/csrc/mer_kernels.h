// mer_kernels.h — internal launch prototypes shared between the .cu files of libmer_b200.so.
// The public C ABI lives in include/mer_b200.h; the structs used here are defined there.
#pragma once
#include <cuda_runtime.h>
#include "../../include/mer_b200.h"

// runtime.cu — optional per-launch CUDA-event timing (bench.py roofline).  klass: MER_GEMM_* for the GEMM
// modes, MER_PROF_* below for the other kernels; work = algorithmic FLOPs or bytes of the launch.
// begin returns a slot (or -1 when profiling is off); end records the closing event.
enum { MER_PROF_F16_SMALL = 3, MER_PROF_CONV_F16 = 4, MER_PROF_ATT_F16 = 10, MER_PROF_ATT_TC = 11, MER_PROF_LAYERNORM = 12, MER_PROF_POSCONV = 13,
       MER_PROF_CONV0 = 14, MER_PROF_ATT_LONG = 15 };
int mer_prof_begin(int klass, double work, cudaStream_t stream);
void mer_prof_end(int slot, cudaStream_t stream);
void mer_prof_pause(int on);  // nest: launches of a composite op (timed as a whole) are not recorded themselves
int mer_cast_f16_launch(const float* in, void* out, long long n, cudaStream_t stream);  // rowwise.cu
int mer_accumulate_launch(const float* x, float* acc, long long n, int init, cudaStream_t stream);  // acc (+)= x

// One-shot per-device state (cudaFuncSetAttribute, the SM count): keyed by the current device so that a process
// driving several GPUs does not reuse the first device's setup.  Not a lock: the C ABI is single-threaded per
// device (mer_b200.h), a repeated cudaFuncSetAttribute is harmless.
struct MerPerDevice {
  bool done[64] = {};
  static int current() {
    int d = 0;
    return (cudaGetDevice(&d) == cudaSuccess && d >= 0 && d < 64) ? d : 0;
  }
  bool needs_setup() const { return !done[current()]; }
  void mark() { done[current()] = true; }
};

// gemm.cu
int mer_gemm_launch(const MerGemmDesc* g, cudaStream_t stream);

// rowwise.cu
int mer_layernorm_launch(const float* x, const float* gamma, const float* beta, float* y,
                         void* y_split, float* acc, long long rows, int dim, float eps, int flags,
                         cudaStream_t stream);

// attention.cu
int mer_attention_launch(const float* qkv, const float* vt, long long vt_ld, float* ctx,
                         const int* cu_seqlens, int n_seq, long long tokens, int max_seqlen, int heads,
                         int flags, cudaStream_t stream);
bool mer_attention_uses_tc(int max_seqlen);  // the tf32 V^T kernel takes this length (needs V^T from the QKV GEMM)
bool mer_attention_legacy();  // MER_ATTENTION_LEGACY set: only the kernel of attention.cu (debug)
// attention_f16.cu: V^T kernels.  out_mode: 0 fp32, 1 tf32-rounded fp32, 2 bf16 hi | lo split rows, 3 fp16
bool mer_attention_f16_supported(int max_seqlen);  // fp16 q | k | V^T, up to 505 tokens
bool mer_attention_f16_long_supported(int max_seqlen);  // 506 .. MER_ATT_LONG_MAX tokens, not under MER_ATTENTION_LEGACY
int mer_attention_f16_long_launch(const void* qkv16, const void* vt16, long long vt_ld, void* ctx, const int* cu_seqlens,
                                  int n_seq, long long tokens, int heads, int max_seqlen, int out_mode, cudaStream_t stream);
int mer_attention_f16_launch(const void* qkv16, const void* vt16, long long vt_ld, void* ctx, const int* cu_seqlens,
                             int n_seq, long long tokens, int heads, int max_seqlen, int out_mode, cudaStream_t stream);
int mer_attention_tc_launch(const float* qkv, const float* vt, long long vt_ld, float* ctx, const int* cu_seqlens,
                            int n_seq, long long tokens, int heads, int max_seqlen, int out_mode, cudaStream_t stream);
// attention_short.cu: the fp16 V^T operands of rows of <= 249 tokens, one CTA per (sequence, head)
bool mer_attention_short_enabled(int max_seqlen);  // 129 .. 208 tokens; MER_ATT_SHORT=1: any <= 249, =0: none
int mer_attention_short_launch(const void* qkv16, const void* vt16, long long vt_ld, void* ctx, const int* cu_seqlens,
                               int n_seq, long long tokens, int heads, int max_seqlen, int out_mode, cudaStream_t stream);

// helpers.cu
int mer_vit_patchify_launch(const uint8_t* frames_bgr, int n_frames, float* a_patches,
                            cudaStream_t stream);
int mer_vit_cls_rows_launch(const float* cls_pos0, float* x, int n_frames, cudaStream_t stream);
int mer_patchify_generic_launch(const uint8_t* frames, int n, int H, int W, int y0, int x0, int size, int patch,
                                int kpad, const float mean[3], const float std[3], float* a, cudaStream_t stream);
int mer_cls_rows_generic_launch(const float* row, float* x, int n_frames, int tokens, int dim, cudaStream_t stream);
int mer_gather_rows_launch(const float* in, long long first, long long step, int n, int dim, float* out,
                           cudaStream_t stream);
int mer_segment_reduce_launch(const float* in, const int* begins, const int* ends, int n_seg,
                              int dim, int mode, float* out, cudaStream_t stream);
int mer_bert_embed_launch(const int* ids, const int* pos_ids, const float* word, const float* pos,
                          const float* type0, const float* gamma, const float* beta, float eps,
                          int tokens, float* out, void* out_split, cudaStream_t stream, int dim = 768);

// hubert_frontend.cu
// lengths (device, optional): ragged batch, row b holds lengths[b] <= L samples; the tail is written as zeros
int mer_wave_normalize_launch(const float* in, float* out, int B, int L, long long ld_in,
                              long long ld_out, cudaStream_t stream, const int* lengths = nullptr);
// conv0 (+ bias) + LayerNorm over the 512 channels + GELU (HubertLayerNormConvLayer), split-bf16 rows out
int mer_hubert_conv0_ln_launch(const float* wave, long long ld_wave, int B, int L, const float* w0,
                               const float* bias, const float* gamma, const float* beta, float* out,
                               long long out_bstride, cudaStream_t stream);
int mer_hubert_conv0_launch(const float* wave, long long ld_wave, int B, int L, const float* w0,
                            const float* gamma, const float* beta, double* stats, float* out,
                            long long out_bstride, int split_out, cudaStream_t stream,
                            const int* t0s = nullptr);  // t0s (device, optional): per-clip frame counts (ragged batch)
// ragged batch: clip b owns rows [b * Tmax, b * Tmax + tb[b]) of a padded [B, Tmax, dim] activation
int mer_zero_tail_rows_f16_launch(void* x16, const int* tb, int B, int Tmax, int dim, cudaStream_t stream);
int mer_pack_rows_launch(const float* padded, const int* cu, int B, int Tmax, int dim, float* packed,
                         cudaStream_t stream);
// posconv.cu
int mer_posconv_launch(const float* x0, const float* wp, const float* bias, const int* cu_seqlens,
                       int n_seq, int max_seqlen, float* x1, cudaStream_t stream);
int mer_iota_offsets_launch(int* offsets, int n_seg, int step, cudaStream_t stream);

// encoder.cu — transformer stack shared by ViT (pre-LN) and HuBERT/BERT (post-LN)
struct MerStackArgs {
  const MerLayerWeights* layers;
  int n_layers;
  int pre_ln;
  int mode;                  // MER_GEMM_TF32 | MER_GEMM_BF16X3 | MER_GEMM_F16, either order (no caller runs post-LN TF32)
  int dim, ffn, heads;       // 0 = 768 / 3072 / 12
  int quick_gelu;            // FC1 activation: x * sigmoid(1.702 x) (CLIP) instead of erf-GELU
  float eps;
  long long tokens;          // total packed tokens (rows of x)
  const int* cu_seqlens;     // device [n_seq+1]
  int n_seq;
  int max_seqlen;
  float* x;                  // [tokens,768] residual stream (in/out)
  float* xn;                 // [tokens,768] scratch (LN out / attention ctx / pre-LN sum)
  float* xs;                 // BF16X3 only: [tokens,768] slots holding the split copy of x
  float* vt;                 // [768, vt_ld] V^T for the V^T attention kernels (or null: attention.cu)
  long long vt_ld;           // >= tokens, multiple of 4
  float* qkv;                // [tokens,2304]
  float* h;                  // [tokens,3072]
  float* acc;                // optional [tokens,768]: sum of the last `acc_last` hidden states
  int acc_last;
  float* opt_hidden;         // optional [(n_layers+1), tokens, 768]
  int hidden0_done;          // caller already wrote opt_hidden[0] (post-LN: the un-rounded LN)
  int long_rows;             // 1 (HuBERT / wav2vec2): rows of 506 .. MER_ATT_LONG_MAX tokens take the fp16 V^T kernel
                             // like the 254 .. 505-token rows; 0: they take the kernel of attention.cu
};
int mer_run_stack(const MerStackArgs& a, cudaStream_t stream);
