/* mer_b200.h — C ABI of libmer_b200.so (H100 / sm_90a only; the b200 in the names is the project's original tag).
 *
 * Drop-in boundary for the MERTools hot path (SURVEY.md §8b): the reference has no FFI; the
 * seam a maintainer would bind is the model-object call
 *     model(x, output_hidden_states=True).hidden_states  ->  readout
 * in MERBench/feature_extraction/{visual/extract_vision_huggingface.py:140-144,
 * audio/extract_audio_huggingface.py:93-100, text/extract_text_huggingface.py:222-231}
 * and the fusion step of MERBench/main-release.py:31-66.  Every function below cites the
 * reference lines it replaces.  INTEGRATION.md shows the ctypes stub on the reference side.
 *
 * Conventions: all pointers are DEVICE pointers owned by the caller unless a parameter is
 * documented as host; `stream` is a cudaStream_t passed as void*; return 0 on success, non-zero
 * on failure with the message available from mer_last_error().  No global state besides the
 * per-thread error string and cached device attributes.  No CPU fallback exists.
 */
#ifndef MER_B200_H_
#define MER_B200_H_

#include <stdint.h>

#if defined(__GNUC__)
#define MER_API __attribute__((visibility("default")))
#else
#define MER_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ---- library ------------------------------------------------------------------------- */
MER_API const char* mer_last_error(void);
MER_API int mer_abi_version(void); /* 4: model structs may only grow at the tail; zero-filled tails = the older behaviour */
/* 0 when the current device is compute capability 9.0 (H100; the library holds sm_90a code only), non-zero (and an
 * error string) otherwise */
MER_API int mer_check_device(void);

/* cumulative number of CUDA kernels this library has launched in this process (bench.py's
 * gpu_launches); CUDA-graph replays are not seen here and are counted by their owner */
MER_API long long mer_launch_count(void);
/* launches so far of the instantiation gemm_kernel<block_n (128 | 256), mode (MER_GEMM_*)>; cluster (1 | 2) and twosm
 * (0 | 1) name CTA-pair forms, which this build does not have (0 launches for cluster 2 or twosm 1); -1 for arguments
 * outside those ranges. */
MER_API long long mer_gemm_variant_launches(int block_n, int mode, int cluster, int twosm);
/* launches so far of gemm_kernel with the epilogue that stages the output in shared memory and stores it with TMA
 * (tma = 1: fp32, tf32 or fp16 output without residual or activation, the out base at out_row0 and its pitches
 * multiples of 16 bytes, V^T if any starting at a multiple of 32 fp32 / 64 fp16 columns) or with the register epilogue
 * (tma = 0: every other descriptor, and all of them under the environment variable MER_GEMM_EPI_TMA=0, read at every
 * launch); -1 for other arguments.  Both write the same bits. */
MER_API long long mer_gemm_epilogue_launches(int tma);
/* per-launch CUDA-event timing (roofline in bench.py): enable(1) starts a fresh recording, enable(0)
 * stops; collect sums duration / algorithmic work / launches of one kernel class since the last
 * enable(1).  Classes: MER_GEMM_* (work = 2*M*N*K flop; MER_GEMM_F16 launches of fewer than 2^17 rows are
 * class 3; 4 = HuBERT conv1 / conv2 as fp16 implicit GEMMs), 10 = fp16 V^T attention, 11 = TF32 V^T
 * attention (work = 4*S^2*64 flop per (sequence, head), S = tokens / n_seq), 12 = LayerNorm, 14 = HuBERT
 * conv0 (work = algorithmic HBM bytes), 13 = HuBERT positional conv (flop). */
MER_API int mer_profile_enable(int on);
MER_API int mer_profile_collect(int mode, double* total_ms, double* total_flops, int* launches);

/* ---- GEMM (nn.Linear / Conv1d-as-GEMM / patch-embed) ---------------------------------- */
enum { MER_EPI_GELU = 1,
       MER_EPI_ROUND_TF32 = 2, /* out (and vt) rounded to tf32 (cvt.rna); excludes MER_EPI_SPLIT_BF16 */
       MER_EPI_SPLIT_BF16 = 4,
       MER_EPI_GELU_LIBM = 8, /* with MER_EPI_GELU (required): libdevice erff instead of the 12-op polynomial */
       MER_EPI_QUICK_GELU = 64, /* x * sigmoid(1.702 x) (CLIP's hidden_act) instead of GELU; excludes MER_EPI_GELU */
       MER_EPI_RELU = 128,    /* max(x, 0), applied AFTER the residual add when there is one (ResNet BasicBlock);
                                 fp32 output, or fp16 output without a residual (OPT's fc1); excludes the GELU flags */
       MER_EPI_GELU_TANH = 256, /* 0.5 x (1 + tanh(0.79788456 x (1 + 0.044715 x^2))) (BLOOM's bloom_gelu_forward),
                                   |error| <= 1e-6; fp32 or fp16 output, optional bias; no residual / split / tf32 /
                                   V^T, excludes the other activations */
       MER_EPI_OUT_F16 = 16,  /* out (and vt, if given) are IEEE fp16 arrays (round-to-nearest, saturating);
                                 ld_out / vt_ld in elements */
       MER_ATT_QKV_F16 = 32   /* mer_attention only: qkv and vt are fp16 arrays (needs vt, vt_ld % 8 == 0, max_seqlen <=
                                 505); ctx in the format the other flags name (fp16, fp32, MER_EPI_ROUND_TF32,
                                 MER_EPI_SPLIT_BF16): attention_f16.cu */ };
/* Arithmetic mode of a GEMM.  TF32: operands are fp32 arrays (pre-rounded to tf32).  BF16X3: every
 * operand value x is stored as a bf16 pair (hi, lo), x = hi + lo to 2^-17; a row of K values (K % 32
 * == 0) occupies the bytes K fp32 values would, as 128-byte groups [32 x hi | 32 x lo]; three bf16
 * MMAs per product (hi*hi + lo*hi + hi*lo) recover ~fp32 accuracy ("split rows" below).
 * F16: operands are IEEE fp16 arrays (A and W), products exact, fp32 accumulate.  fp16 carries the
 * same 10 mantissa bits as tf32, so a GEMM on fp16-rounded operands equals the TF32 GEMM on the same
 * values (|x| in [6.1e-5, 65504]; smaller magnitudes lose at most 3e-8 absolute) at twice the
 * tensor-pipe rate and half the operand bytes.  K_inner % 64 == 0; all A strides in fp16 elements. */
enum { MER_GEMM_TF32 = 0, MER_GEMM_BF16X3 = 1, MER_GEMM_F16 = 2 };

typedef struct MerGemmEpilogue {
  const float* bias; /* [N] or NULL; 8-byte aligned */
  const float* res;  /* residual rows or NULL; 8-byte aligned */
  float* out;        /* 8-byte aligned (4-byte for an fp16 out) */
  long long out_bstride; /* out row = b*out_bstride + out_row0 + m */
  long long out_row0;
  long long res_bstride; /* res row = b*res_bstride + res_row0 + m */
  long long res_row0;
  int ld_out; /* floats */
  int ld_res;
  int flags;     /* MER_EPI_* */
  int split_off; /* reserved (0) */
  /* optional transposed side output: columns n >= vt_col0 are written as vt[(n - vt_col0) * vt_ld +
   * out_row] INSTEAD of out[out_row, n] (the QKV GEMM hands V^T, keys contiguous, to the V^T
   * attention kernel); with vt, vt_col0 must be even and in [0, N) */
  float* vt;
  long long vt_ld;
  int vt_col0;
} MerGemmEpilogue;

/* A[b, m, tap*K_inner + c] = base[b*a_batch_stride + (m + tap / P)*a_row_stride +
 *                                 (tap % P)*a_phase_stride + c]        (element strides)
 * Plain row-major A[M,K]: taps = 1, P = 1, K_inner = K, batches = 1, a_row_stride = K.
 * Conv1d(kernel k, stride s) over time-major activations x[b, tau, c]:
 *   taps = k, P = s, K_inner = C_in, a_phase_stride = C_in, a_row_stride = s*C_in.           */
typedef struct MerGemmDesc {
  const float* A;
  const float* W; /* [N, taps*K_inner] row-major (nn.Linear layout) */
  int rows_per_batch;
  int a_rows_dim; /* addressable row groups per batch entry (>= rows_per_batch + (taps-1)/P) */
  int batches;
  int N;
  int K_inner;
  int taps;
  int P;
  long long a_phase_stride;
  long long a_row_stride;
  long long a_batch_stride;
  int force_block_n; /* 0 = auto, 128 or 256 */
  int mode;          /* MER_GEMM_TF32 | MER_GEMM_BF16X3 (A strides in 4-byte slots) | MER_GEMM_F16 (A strides in
                        2-byte elements) */
  int cluster;       /* reserved: CTA-pair tiles; every value runs single-CTA tiles on sm_90a */
  /* grouped-convolution support (the HuBERT positional conv runs as a block-diagonal GEMM):
   * a_row0     : added to every A row index (may be negative); rows outside [0, a_rows_dim) of a batch
   *              entry read as zero -- the conv's zero padding.
   * a_cols     : addressable A columns per row (0 = K_inner).
   * a_col_group: when > 0, the K_inner-wide column window of output column block j starts at
   *              floor(j * block_n / a_col_group) * a_col_group (block_n = force_block_n, required);
   *              columns beyond a_cols read as zero.  W holds the matching windowed weights. */
  int a_row0;
  int a_cols;
  int a_col_group;
  MerGemmEpilogue ep;
} MerGemmDesc;

/* wgmma GEMM with fused epilogue.  Replaces torch nn.Linear / nn.Conv1d calls inside
 * HF ViTLayer / HubertEncoderLayer / BertLayer reached from the reference extractors. */
MER_API int mer_gemm(const MerGemmDesc* desc, void* stream);
/* fp32 [rows, K] -> split rows (same byte size, K % 32 == 0); used on weights at load time */
MER_API int mer_split_bf16(const float* in, void* out, long long rows, int K, void* stream);

/* ---- row-wise kernels ------------------------------------------------------------------ */
enum { MER_LN_ROUND_TF32 = 1, MER_LN_ACC_INIT = 2, MER_LN_ACC_ADD = 4,
       MER_LN_OUT_F16 = 8, /* y is an fp16 array (the MER_GEMM_F16 operand) */
       MER_LN_GELU = 16,   /* GELU(erf) after the affine (HubertLayerNormConvLayer) */
       MER_LN_SPLIT_F16 = 32, /* y_split is an fp16 array (the MER_GEMM_F16 operand) written NEXT TO the fp32 y:
                                the post-LN stacks keep y as their residual stream */
       MER_LN_PAD = 64 /* dim is the valid width of rows padded to the next multiple of 128 (x, y, y_split, acc, gamma
                          and beta all have the padded width): mean and variance over the first dim columns only, and
                          every output (y, y_split, acc) is written as exactly 0 in the pad columns, whatever x, gamma
                          and beta hold there (albert_chinese_tiny: 312 valid columns in 384).  Always the default
                          (round-2) kernel form. */ };
/* y = LayerNorm(x) * gamma + beta over the last dim (128, 384, 512, 768, 1024, 1280 or 1536; with MER_LN_PAD, any dim
 * whose next multiple of 128 is one of them).  y (fp32, tf32-rounded when
 * MER_LN_ROUND_TF32) and y_split (bf16 hi|lo rows, the BF16X3 GEMM operand) are both optional;
 * at least one must be given.  Optional side buffer acc
 * (same shape): acc = y (ACC_INIT) or acc += y (ACC_ADD) — the "sum of the last four hidden
 * states" readout of extract_audio_huggingface.py:98 / extract_text_huggingface.py:226.  acc and y_split take the fp32
 * value before y's tf32 / fp16 rounding; ACC_INIT wins over ACC_ADD; without either flag acc is not touched.  fp16
 * outputs saturate at +-65504.  y == x and y_split == x are allowed (not an fp16 y); rows <= 0 is a no-op. */
MER_API int mer_layernorm(const float* x, const float* gamma, const float* beta, float* y,
                          void* y_split, float* acc, long long rows, int dim, float eps, int flags,
                          void* stream);

/* in-place round-to-nearest fp32 -> tf32 (weights at load time) */
MER_API int mer_round_tf32(float* x, long long n, void* stream);

/* ---- attention ------------------------------------------------------------------------- */
/* softmax(Q K^T / 8) V per (sequence, head); head_dim 64.  qkv is [tokens, 3*heads*64] with
 * Q | K | V column blocks, sequences packed back to back, cu_seqlens[n_seq+1] (device, int32),
 * tokens = cu_seqlens[n_seq] (host copy, sizes the TMA descriptors).  vt (optional): V^T, [heads*64,
 * vt_ld] with vt[d, token] = V[token, d] (vt_ld >= tokens, multiple of 4; of 8 for fp16), as written by mer_gemm's
 * transposed side output.  Three routes, chosen from flags, vt and max_seqlen (not from the lengths in cu_seqlens):
 *  1. MER_ATT_QKV_F16: qkv and vt are fp16 (attention_f16.cu: fp16 MMAs, half the traffic); vt is required and
 *     max_seqlen <= 505, anything else is refused.  ctx in any of the four forms below.
 *  2. fp32 qkv, vt given and max_seqlen <= 253: the tf32 V^T kernel; the V columns of qkv are not read.  ctx in any of
 *     the four forms.
 *  3. fp32 qkv otherwise (no vt, or max_seqlen >= 254; every call when the environment variable MER_ATTENTION_LEGACY
 *     is set at the first call): the kernel that reads V from qkv (attention.cu), any length; vt is not read.
 *     ctx fp32, tf32-rounded or split; MER_EPI_OUT_F16 is refused.
 * ctx is [tokens, heads*64].  flags: none = fp32; MER_EPI_ROUND_TF32 rounds ctx for a TF32 out-proj GEMM;
 * MER_EPI_SPLIT_BF16 writes ctx as bf16 hi|lo rows for a BF16X3 out-proj GEMM; MER_EPI_OUT_F16 writes ctx as fp16 for
 * an F16 out-proj GEMM (OUT_F16 wins over SPLIT_BF16, which wins over ROUND_TF32).  n_seq <= 65535, heads <= 65535;
 * on route 3 n_seq <= 0 or max_seqlen <= 0 is a no-op and the rows of a sequence beyond max_seqlen are not written.
 * Replaces HF eager/sdpa attention (modeling_vit.py:171-196, modeling_hubert.py:262-345). */
MER_API int mer_attention(const float* qkv, const float* vt, long long vt_ld, float* ctx,
                          const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen,
                          int heads, int flags, void* stream);
/* mer_attention's V^T route (routes 1 and 2) at head_dim 32 or 64 with an explicit score scale: softmax(scale Q K^T) V
 * (HF AlbertSdpaAttention / eager attention: scale 1 / sqrt(hidden / heads)).  qkv [tokens, 3 * heads * head_dim] with
 * Q | K column blocks (V columns not read), vt [heads * head_dim, vt_ld] (vt_ld >= tokens, multiple of 8 for fp16 / 4
 * for fp32), ctx [tokens, heads * head_dim].  flags: MER_ATT_QKV_F16 (fp16 qkv / vt) or none (tf32-rounded fp32), plus
 * MER_EPI_OUT_F16 / MER_EPI_SPLIT_BF16 / MER_EPI_ROUND_TF32 for ctx as in mer_attention.  Rows of up to 512 tokens, on
 * both operand formats.  A head zero-padded to 32 columns (ALBERT's 26) gives the unpadded result when scale is that of
 * the unpadded head, and zero ctx in the pad columns.  head_dim 64 at scale 0.125 runs what mer_attention runs for rows
 * it accepts (bit for bit).  Refused before any launch with a "mer_attention_hd:" message: head_dim other than 32 / 64,
 * scale outside (0, 1] or NaN, a NULL operand, other flags, a V^T pitch that is too small or misaligned, max_seqlen
 * outside 1 .. min(512, tokens), heads or n_seq outside 1 .. 65535.  attention_f16.cu. */
MER_API int mer_attention_hd(const void* qkv, const void* vt, long long vt_ld, void* ctx, const int32_t* cu_seqlens,
                             int n_seq, long long tokens, int max_seqlen, int heads, int head_dim, float scale,
                             int flags, void* stream);

/* Longest row of mer_attention_long, and of the HuBERT / wav2vec2 stacks' fp16 V^T attention (82 s of audio; a 60 s
 * clip is 2,999 frames).  Longer rows of those stacks take the kernel of attention.cu (route 3 above). */
#define MER_ATT_LONG_MAX 4096
/* mer_attention's fp16 route (route 1) for rows of up to MER_ATT_LONG_MAX tokens: qkv fp16 [tokens, 3 * heads * 64]
 * (V columns not read), vt fp16 [heads * 64, vt_ld], ctx [tokens, heads * 64] in the format the flags name
 * (MER_EPI_OUT_F16, MER_EPI_SPLIT_BF16, MER_EPI_ROUND_TF32 or none = fp32).  Rows of up to 505 tokens run exactly what
 * mer_attention runs; longer ones the same tiled kernel over more 64-key tiles (fp16 P, fp32 softmax statistics).  The
 * HuBERT / wav2vec2 stacks route their rows of 506 .. MER_ATT_LONG_MAX tokens here (not under MER_ATTENTION_LEGACY).
 * Refused before any launch with a "mer_attention_long:" message: a NULL operand, other flags, tokens outside
 * 1 .. 2^31 - 1, a V^T pitch below tokens or not a multiple of 8, max_seqlen outside 1 .. min(MER_ATT_LONG_MAX,
 * tokens), heads or n_seq outside 1 .. 65535.  attention_f16.cu. */
MER_API int mer_attention_long(const void* qkv, const void* vt, long long vt_ld, void* ctx, const int32_t* cu_seqlens,
                               int n_seq, long long tokens, int max_seqlen, int heads, int flags, void* stream);

/* ---- segment reduce (readouts) ------------------------------------------------------------ */
enum { MER_SEG_SUM = 0, MER_SEG_MEAN = 1 };
/* out[s, :] = sum or mean of in[begins[s] : ends[s], :] (dim % 4 == 0; begins/ends device int32,
 * n_seg entries each; for back-to-back segments pass offsets and offsets+1).  Empty segments give zeros (extract_text_huggingface.py:236-249 writes zeros
 * for an empty sentence).  Replaces hidden_states[-1].sum(dim=1) / np.mean(axis=0)
 * (extract_vision_huggingface.py:144,187-188; extract_audio_huggingface.py:105-108). */
MER_API int mer_segment_reduce(const float* in, const int32_t* begins, const int32_t* ends, int n_seg,
                               int dim, int mode, float* out, void* stream);

/* ---- transformer encoder stack shared by the three modalities ----------------------------------- */
/* GEMM weights (w_*) are tf32-rounded fp32 [N,K] for a MER_GEMM_TF32 stack and split bf16
 * split rows for a MER_GEMM_BF16X3 stack (ViT: TF32; HuBERT/BERT: BF16X3). */
typedef struct MerLayerWeights {
  const float* ln1_g; /* ViT: layernorm_before | HuBERT: layer_norm | BERT: attention.output.LayerNorm */
  const float* ln1_b;
  const float* w_qkv; /* [2304, 768] = rows Q | K | V, tf32-rounded */
  const float* b_qkv; /* [2304] */
  const float* w_o;   /* [768, 768] */
  const float* b_o;
  const float* ln2_g; /* ViT: layernorm_after | HuBERT: final_layer_norm | BERT: output.LayerNorm */
  const float* ln2_b;
  const float* w_fc1; /* [3072, 768] */
  const float* b_fc1;
  const float* w_fc2; /* [768, 3072] */
  const float* b_fc2;
} MerLayerWeights;
/* gamma / beta of one LayerNorm (device pointers); the per-layer FFN norms of the EVA02 tower */
typedef struct MerNormWeights {
  const float* g;
  const float* b;
} MerNormWeights;

/* ---- frame resize (visual preprocessing) ------------------------------------------------------- */
/* PIL.Image.resize((OW, OH), BILINEAR) on uint8 [n, H, W, 3] frames, bit-exact: the resize step of HF
 * ViTImageProcessor (extract_vision_huggingface.py:137-138) for faces that are not 224x224 already
 * (OpenFace crops are 112x112).  Horizontal pass, then vertical pass, uint8 in between.  workspace:
 * mer_resize_workspace_bytes(...) bytes (0 when only one axis changes). */
MER_API long long mer_resize_workspace_bytes(int n, int H, int W, int OH, int OW);
MER_API int mer_resize_bilinear_u8(const uint8_t* in, int n, int H, int W, uint8_t* out, int OH, int OW,
                                   void* workspace, void* stream);
/* same with a filter choice: 0 = BILINEAR, 1 = BICUBIC (Pillow's a = -0.5 cubic; HF CLIPImageProcessor) */
MER_API int mer_resize_u8(const uint8_t* in, int n, int H, int W, uint8_t* out, int OH, int OW, int filter,
                          void* workspace, void* stream);
/* cv2.resize(frame, (out_w, out_h)) with the default INTER_LINEAR, bit-exact against OpenCV 4.13 (fixed-point
 * coefficients, border rules and the 2x-downscale area path of imgproc/src/resize.cpp): what the EmoNet extractor's
 * DataAugmentor does to every face (emonet/data_augmentation.py:77).  frames uint8 [n, h, w, 3] -> [n, out_h, out_w, 3]. */
MER_API int mer_resize_cv2_linear_u8(const uint8_t* frames, int n, int h, int w, uint8_t* out, int out_h, int out_w,
                                     void* stream);

/* ---- ViT-B/16 frame encoder (visual) ------------------------------------------------------------ */
typedef struct MerVitModel {
  int n_layers;        /* 12 */
  float ln_eps;        /* 1e-12 */
  int gemm_mode;       /* MER_GEMM_F16 (layer weights w_* are fp16 [N,K]) or MER_GEMM_TF32 (tf32-rounded fp32) */
  const float* patch_w;   /* [768, 768]  conv weight flattened (c, ph, pw), tf32-rounded */
  const float* patch_b;   /* [768] */
  const float* cls_pos0;  /* [768]  cls_token + position_embeddings[0] */
  const float* pos_rest;  /* [196, 768] position_embeddings[1:] */
  const MerLayerWeights* layers; /* host array of n_layers entries (device pointers inside) */
} MerVitModel;

/* bytes of caller-provided device workspace for n_frames frames */
MER_API long long mer_vit_workspace_bytes(int n_frames);

/* frames: uint8 [n_frames, 224, 224, 3] BGR (the reference's openface_face/<vid>/<vid>.npy layout).
 * Does, on the device: BGR->RGB, x/255, (x-.5)/.5 (HF ViTImageProcessor as invoked at
 * extract_vision_huggingface.py:137-138), the 12-layer pre-LN ViT forward (HF modeling_vit.py),
 * and the readout hidden_states[-1].sum(dim=1) (extract_vision_huggingface.py:143-144).
 * out_frame_feats: [n_frames, 768].  opt_hidden: NULL or [(n_layers+1), n_frames*197, 768] to
 * receive every hidden state (parity tests). */
MER_API int mer_vit_forward(const MerVitModel* model, const uint8_t* frames_bgr, int n_frames,
                            void* workspace, long long workspace_bytes, float* out_frame_feats,
                            float* opt_hidden, void* stream);

/* ---- CLIP vision tower (clip-vit-base-patch32 / clip-vit-large-patch14) ---------------------------- */
/* model.get_image_features(pixel_values) of the reference's CLIP branch (extract_vision_huggingface.py:
 * 114-122; HF modeling_clip.py): patch embedding (no bias) + class / position embeddings, pre_layrnorm,
 * pre-LN layers with quick_gelu, post_layernorm of the class token, visual_projection. */
typedef struct MerClipVisionModel {
  int n_layers;
  float ln_eps;        /* 1e-5 */
  int hidden, ffn, heads, patch, image, proj_dim; /* 768/3072/12/32/224/512 or 1024/4096/16/14/224/768 */
  int kpad;            /* columns of patch_w: 3*patch*patch rounded up to a multiple of 32 (zero-filled) */
  int gemm_mode;       /* MER_GEMM_F16 (<= 249 tokens per frame) or MER_GEMM_TF32: format of the layer weights */
  float mean[3], std[3];  /* CLIPImageProcessor image_mean / image_std (RGB) */
  const float* patch_w;   /* [hidden, kpad] conv weight flattened (c, ph, pw), tf32-rounded */
  const float* cls_pos0;  /* [hidden] class_embedding + position_embedding[0] */
  const float* pos_rest;  /* [(image/patch)^2, hidden] position_embedding[1:] */
  const float* pre_ln_g;  /* pre_layrnorm */
  const float* pre_ln_b;
  const float* post_ln_g; /* post_layernorm */
  const float* post_ln_b;
  const float* proj_w;    /* visual_projection.weight [proj_dim, hidden], tf32-rounded */
  const MerLayerWeights* layers;
  /* 0 (zero-initialised): CLIP as described above.  MER_VISION_DINOV2 (1): HF Dinov2Model (dinov2-large,
   * extract_vision_huggingface.py:135-145) on the same tower: no pre_layrnorm (pre_ln_g NULL), erf GELU, LayerScale
   * folded into the out-proj / FC2 weights and the patch-conv bias into pos_rest by the loader, position table already
   * interpolated to the image grid; out_embeds [n_frames, hidden] = sum over the tokens of the LAST LAYER's output
   * (hidden_states[-1], before Dinov2Model.layernorm); post_ln_* / proj_w unused, proj_dim = hidden. */
  /* MER_VISION_EMBED_ONLY (2): stop after the embeddings; out_embeds [n_frames * tokens, hidden] = class row
   * (cls_pos0) + patch rows (patch conv + pos_rest) = hidden_states[0] of a model whose layers the host orchestrates
   * (data2vec-vision: relative position bias in attention, extract/data2vec_vision.py); layers / n_layers unused. */
  /* MER_VISION_EVA02 (3): timm Eva (eva02_base_patch14_224, the EVACLIP_VIT branch of the visual extractor) on the same
   * tower: no pre_layrnorm (pre_ln_g NULL), the patch-conv bias folded into pos_rest, q_bias | 0 | v_bias as b_qkv; in
   * every layer the 2D rotary embedding below on the q | k of the patch rows (the class row is not rotated), and the
   * FFN x + fc2(LN(silu(fc1_g h) * fc1_x h)) with w_fc1 / b_fc1 = rows fc1_g | fc1_x ([2 ffn, hidden]), w_fc2 [hidden,
   * ffn] and the LN of ffn_norms (eps ln_eps).  out_embeds [n_frames, hidden] = post_ln (fc_norm) of the mean over the
   * patch rows of the last layer's output; proj_w unused, proj_dim = hidden.  Refused before any launch: a NULL table or
   * norm array, NULL post_ln_*, rope_rows other than (image / patch)^2, ffn > 3 hidden, gemm_mode MER_GEMM_BF16X3.
   * Attention at 257 tokens runs on fp16 q | k | V^T in both operand formats, so the rotation is always on fp16. */
  int variant;
  const float* rope_cos;  /* MER_VISION_EVA02: [rope_rows, 32] fp32 cos of the pair angles of each patch row */
  const float* rope_sin;  /* (see mer_rope2d_f16); 16-byte aligned */
  int rope_rows;
  const MerNormWeights* ffn_norms; /* MER_VISION_EVA02: host array of n_layers entries (mlp.norm) */
} MerClipVisionModel;
#define MER_VISION_CLIP 0
#define MER_VISION_DINOV2 1
#define MER_VISION_EMBED_ONLY 2
#define MER_VISION_EVA02 3

/* ---- the EVA02 kernels (csrc/eva02.cu), run by the MER_VISION_EVA02 tower ---- */
/* timm RotaryEmbeddingCat / apply_rot_embed_cat, in place on the q | k columns [0, 2 * heads * 64) of fp16 rows qkv16
 * [tokens, ld]: tokens are whole frames of tokens_per_frame rows whose first `prefix` rows are left alone; row j >=
 * prefix of a frame uses table row p = j - prefix, and for every q / k head and pair i < 32,
 * (x[2i], x[2i+1]) -> (x[2i] c - x[2i+1] s, x[2i+1] c + x[2i] s), c / s = cos_t / sin_t[p * 32 + i] (fp32, built on the
 * host), computed in fp32 and rounded once.  Columns from 2 * heads * 64 on (V) are not touched.  Refused before any
 * launch: a NULL operand, head_dim other than 64, ld < 2 * heads * 64 or not a multiple of 4, a misaligned operand,
 * tokens not a multiple of tokens_per_frame, table_rows != tokens_per_frame - prefix. */
MER_API int mer_rope2d_f16(void* qkv16, long long ld, long long tokens, int tokens_per_frame, int prefix, int heads,
                           int head_dim, const float* cos_t, const float* sin_t, int table_rows, void* stream);
/* timm SwiGLU with its norm (Eva's scale_mlp): in fp32 [rows, 2 * hidden] = rows fc1_g | fc1_x of the FC1 output;
 * out [rows, hidden] = LayerNorm(silu(g) * x) * gamma + beta, mean and centred variance in fp32 over the product kept on
 * chip; out fp16 (out_f16, the MER_GEMM_F16 operand of fc2) or tf32-rounded fp32.  Refused before any launch: hidden
 * not a multiple of 128 or above 4096, a NULL operand, out == in, rows outside 1 .. 2^31 - 1. */
MER_API int mer_swiglu_ln(const float* in, const float* gamma, const float* beta, float eps, void* out, long long rows,
                          int hidden, int out_f16, void* stream);

MER_API long long mer_clip_vision_workspace_bytes(const MerClipVisionModel* model, int n_frames);

/* frames: uint8 [n_frames, H, W, 3] BGR already resized so that the shorter edge is `image` (mer_resize_u8,
 * bicubic); the image x image window at (crop_y0, crop_x0) is the processor's center crop.  Does BGR->RGB,
 * x/255, (x - mean) / std, the tower and the projection.  out_embeds: [n_frames, proj_dim].
 * opt_hidden: NULL or [(n_layers+1), n_frames*tokens, hidden] (hidden state 0 = pre_layrnorm output). */
MER_API int mer_clip_vision_forward(const MerClipVisionModel* model, const uint8_t* frames_bgr, int n_frames,
                                    int H, int W, int crop_y0, int crop_x0, void* workspace,
                                    long long workspace_bytes, float* out_embeds, float* opt_hidden, void* stream);

/* ---- ResNet-18 frame encoder (the reference's ImageNet CNN extractor) ------------------------------- */
/* One convolution with its BatchNorm folded in (eval mode): w' = w * gamma / sqrt(var + eps),
 * b' = beta - mean * gamma / sqrt(var + eps).  w: fp16 [cout_pad, kpad] in (ky, kx, c) order, rows >= cout and
 * columns >= k*k*cin zero; b: fp32 [cout_pad].  cout_pad = max(cout, 128); kpad = k*k*cin (192 for conv1). */
typedef struct MerResnetConv {
  const void* w;
  const float* b;
  int cin, cout, cout_pad, k, stride, pad, kpad;
} MerResnetConv;

/* torchvision.models.resnet18 without fc, in module order: conv1; layer1.{0,1}.{conv1,conv2};
 * layerX.0.{conv1,conv2,downsample}, layerX.1.{conv1,conv2} for X = 2..4  (20 convolutions). */
typedef struct MerResnet18Model {
  MerResnetConv convs[20];
  float mean[3], std[3]; /* transforms.Normalize (RGB): 0.485 0.456 0.406 / 0.229 0.224 0.225 */
} MerResnet18Model;

MER_API long long mer_resnet18_workspace_bytes(int n_frames);
/* frames: uint8 [n_frames, 224, 224, 3] BGR (resize other sizes first: transforms.Resize((224, 224)) is PIL
 * bilinear = mer_resize_bilinear_u8).  Does BGR->RGB, ToTensor, Normalize, the network up to the global average
 * pool (extract_imagenet_embedding.py:47-55, dataset.py:40-47).  out_feats: [n_frames, 512]. */
MER_API int mer_resnet18_forward(const MerResnet18Model* model, const uint8_t* frames_bgr, int n_frames,
                                 void* workspace, long long workspace_bytes, float* out_feats, void* stream);

/* ---- table-driven CNN executor: frame-level CNN extractors as chains of conv (+ folded BatchNorm, + residual,
 * + ReLU), max-pools, crops / channel slices, gates, per-channel affines, upsample-adds and average pools over up to
 * 24 NHWC fp32 activation buffers.
 * Users: resnet50_ferplus_dag / senet50_ferplus_dag up to conv5_3_3x3_relu + AvgPool2d(7)
 * (MERBench/feature_extraction/visual/extract_ferplus_embedding.py:81-115, default --layer_name;
 * pytorch-benchmarks/model/resnet50_ferplus_dag.py:178-355), MA-Net's 1024-d embedding
 * (extract_manet_embedding.py:31-41; manet/model/manet.py:222-270) and EmoNet's 256-d embedding
 * (extract_emonet_embedding.py:22-33; emonet/models/emonet.py:173-222). */
enum { MER_CNN_STEM = 0,    /* dst = act(conv(frames)): 7x7 / 2 / pad 3 on the uint8 input, preprocessing fused */
       MER_CNN_CONV = 1,    /* dst = act(conv(src[..., p0 : p0 + cin]) [+ res]); dst may equal res (in-place update) */
       MER_CNN_MAXPOOL = 2, /* dst = MaxPool2d(3, 2, pad, ceil_mode)(src), windows clipped to the image */
       MER_CNN_GAP = 3,     /* out_feats[:, p0 : p0 + C] (+)= mean over H x W of src / max(p2, 1); p1 != 0 accumulates */
       MER_CNN_SE = 4,      /* squeeze-and-excitation block end (senet50_ferplus_dag): dst = relu(g * src + res),
                               g[n, c] = sigmoid(up(relu(down(mean over H x W of src)))); conv = index of the
                               "down" layer, k = index of the "up" layer: convs entries with k = 1 whose w is a
                               PLAIN fp32 [cout, cin] matrix (not a GEMM operand) and b an fp32 [cout] bias */
       MER_CNN_CROP = 5,    /* dst = src[:, p0 : p0 + p2, p1 : p1 + p3, :] */
       MER_CNN_SHAPE = 6,   /* declares dst as an [H, W] map like src with p0 channels (filled by SLICE ops) */
       MER_CNN_SLICE = 7,   /* dst[..., p1 : p1 + p2] = f(src[..., p0 : p0 + p2]) [+ res[..., p3 : p3 + p2]];
                               relu = 1: f = ReLU; relu = 2: ReLU of the sum */
       MER_CNN_AFFINE = 9,  /* dst = act(src[..., p0 : p0 + C] * a + b) per channel (a pre-activation BatchNorm): conv = an
                               entry whose w is a plain fp32 [C] scale and b the [C] shift, C = its cout; relu = ReLU */
       MER_CNN_UPADD = 10,  /* dst = res + nearest x2 upsample of src (res is [2H, 2W]); dst may equal res */
       MER_CNN_MASKMUL = 11,/* dst[..., p1 : p1 + p2] = src[..., p0 : p0 + p2] * sum over the first p3 channels of res */
       MER_CNN_CBAM = 8 };  /* MA-Net AttentionBlock end: dst = relu(CBAM(src) + res) on maps of <= 64 positions;
                               conv = ChannelGate.mlp.1, p0 = ChannelGate.mlp.3 (plain fp32 dense layers as for SE),
                               p1 = the SpatialGate 7x7 conv: w plain fp32 [2 * 49] with its BatchNorm folded, b [1] */
typedef struct MerCnnOp {
  int kind;  /* MER_CNN_* */
  int conv;  /* STEM / CONV / SE / CBAM: index into convs */
  int src, dst, res; /* buffer indices 0..23; res = -1 for none */
  int relu;  /* STEM / CONV: ReLU (after the residual add); SLICE: see above */
  int k, stride, pad, ceil_mode; /* MAXPOOL (3 / 2 / pad / ceil, or k = 2: plain 2x2 / 2); SE: k = the "up" layer */
  int p[4];  /* op-specific parameters (see the enum) */
} MerCnnOp;
typedef struct MerCnnModel {
  const MerResnetConv* convs; /* BatchNorm folded; w in the layout of gemm_mode: fp16 [cout_pad, kpad] (stem kpad
                                 192) or split bf16 (stem kpad 160), rows in (ky, kx, cin) order */
  int n_convs;
  const MerCnnOp* ops;
  int n_ops;
  int gemm_mode;       /* MER_GEMM_F16 or MER_GEMM_BF16X3 */
  int in_h, in_w;      /* frames are uint8 [n, in_h, in_w, 3] BGR (resize / crop beforehand) */
  float scale;         /* x = (pix * scale - mean[c]) / std[c] in RGB order: 1/255 (ToTensor) or 1 (ToTensor * 255) */
  float mean[3], std[3];
  int feat_dim;        /* width of out_feats (the GAP ops fill column ranges of it) */
} MerCnnModel;

MER_API long long mer_cnn_workspace_bytes(const MerCnnModel* model, int n_frames); /* -1: bad model (mer_last_error) */
MER_API int mer_cnn_forward(const MerCnnModel* model, const uint8_t* frames_bgr, int n_frames, void* workspace,
                            long long workspace_bytes, float* out_feats, void* stream);

/* ---- VGGish audio embedding network (MERBench/feature_extraction/audio/vggish/vggish_slim.py:37-100, called by
 * extract_vggish_embedding.py:30-49 through the TF graph tensors vggish/input_features -> vggish/embedding).
 * convs: conv1, conv2, conv3_1, conv3_2, conv4_1, conv4_2 (3x3, 'SAME', ReLU) in MerResnetConv structs whose w is
 * a SPLIT-BF16 (MER_GEMM_BF16X3) [cout_pad, kpad] matrix, rows in (ky, kx, cin) order = the TF HWIO variable
 * transposed to [O, H, W, I]; conv1: cin 1, kpad 32, cout_pad 128.  fc_w: split-bf16 [N, K] (= the TF [K, N]
 * variable transposed) for fc1_1 (K 12288 = the NHWC flatten of [6, 4, 512]), fc1_2 (4096 x 4096) and fc2
 * (128 x 4096); fc_b fp32 [N]. */
typedef struct MerVggishModel {
  MerResnetConv convs[6];
  const void* fc_w[3];
  const float* fc_b[3];
} MerVggishModel;

MER_API long long mer_vggish_workspace_bytes(int n_examples);
/* examples: fp32 [n_examples, 96, 64] log-mel patches (mer_logmel + the framing of vggish_input.py:37-82);
 * out_embeddings: fp32 [n_examples, 128] = the 'vggish/embedding' tensor (ReLU output of fc2, no PCA
 * post-processing: the reference script saves it as is). */
MER_API int mer_vggish_forward(const MerVggishModel* model, const float* examples, int n_examples, void* workspace,
                               long long workspace_bytes, float* out_embeddings, void* stream);

/* ---- HuBERT-base audio encoder ------------------------------------------------------------------ */
typedef struct MerHubertModel {
  int n_layers;  /* 12 (>= 4 for the readout that sums the last four hidden states; see `readout`) */
  float ln_eps;  /* 1e-5 */
  const float* conv0_w;    /* [512, 10] */
  const float* gn_g;       /* GroupNorm(512 groups) affine, [512] */
  const float* gn_b;
  const float* conv_w[6];  /* conv1..6, [512, k*512] laid out [out][tap][in], split bf16 (BF16X3) */
  const float* fp_ln_g;    /* feature_projection.layer_norm [512] */
  const float* fp_ln_b;
  const float* fp_w;       /* [768, 512] split bf16 (BF16X3) */
  const float* fp_b;
  const float* pos_w;      /* [16][128][48][48] = [group][tap][out][in], weight-norm folded, tf32 */
  const void* pos_w_bd;    /* optional fp16 [768][128 * 320]: the same weights as a windowed block-diagonal
                              matrix (window of output block j starts at channel floor(256 j / 48) * 48), which
                              runs the positional conv through mer_gemm (MER_GEMM_F16); NULL = mma.sync kernel */
  const float* pos_b;      /* [768] */
  const float* enc_ln_g;   /* encoder.layer_norm */
  const float* enc_ln_b;
  const MerLayerWeights* layers;
  /* ---- model family (zero-initialised fields = HuBERT-base / wav2vec2-base) ----
   * hubert-large / chinese-hubert-large / wav2vec2-large-lv60 (extract_audio_huggingface.py:21,27,29):
   * hidden 1024, 16 heads, FFN 4096, feat_extract_norm="layer" (every conv followed by LayerNorm over its 512
   * channels instead of GroupNorm on conv0; conv biases), do_stable_layer_norm (pre-LN layers,
   * encoder.layer_norm applied after the last layer; hidden states taken before each layer). */
  int hidden;              /* 0 = 768; 768 or 1024 */
  int ffn;                 /* 0 = 3072 */
  int heads;               /* 0 = 12; hidden / 64 */
  int feat_norm_layer;     /* 1: LayerNorm after every conv (conv_ln_*), conv biases (conv_b) */
  int stable_layer_norm;   /* 1: pre-LN encoder (HubertEncoderStableLayerNorm) */
  const float* conv_b[7];      /* conv biases [512] (feat_norm_layer) */
  const float* conv_ln_g[7];   /* per-conv LayerNorm affine [512] (feat_norm_layer) */
  const float* conv_ln_b[7];
  int pos_window;          /* K window of pos_w_bd (0 = 320; 256 for 64-channel groups) */
  const MerLayerWeights* layers_f16; /* optional (stable_layer_norm only): the same layers with fp16 GEMM weights;
                              when given, clips of <= 249 frames run the pre-LN stack on fp16 operands
                              (MER_GEMM_F16 + the fp16 attention), longer ones stay BF16X3 */
  /* ---- data2vec-audio (Data2VecAudioModel, extract_audio_huggingface.py:19-20): instead of the single k = 128
   * positional conv, a chain of n_pos_layers grouped convs (pos_taps = 19 taps, padding 9, 16 groups, bias), each
   * followed by an affine-free LayerNorm (eps 1e-5) and GELU; the chain's output is added to its input once.
   * Used with feat_norm_layer = 1 (bias-free convs: conv_b NULL), stable_layer_norm = 0.  0 = classic conv. */
  int n_pos_layers;            /* 0, or up to 8 */
  int pos_taps;                /* odd kernel size of the chain's convs (19) */
  const void* pos_layers_w[8]; /* fp16 windowed block-diagonal matrices [hidden][pos_taps * pos_window] (as pos_w_bd) */
  const float* pos_layers_b[8];/* [hidden] */
  const float* ln_ones;        /* [hidden] ones / zeros: the affine of the affine-free LayerNorms */
  const float* ln_zeros;
  /* ---- operand format of the first convolutions (group-norm feature encoder only; NULL = BF16X3 as conv3..6) ----
   * conv_w_f16[0]: conv1's weights as fp16 [512, 3 * 512] ([out][tap][in]): conv0 then writes fp16 rows and conv1 runs
   * as one MER_GEMM_F16 product instead of three bf16 MMAs; conv_w_f16[1] (needs [0]): the same for conv2 (conv1 then
   * writes fp16 rows, conv2 split-bf16 rows for conv3).  conv1 + conv2 are 77 % of the conv stack's flops; emulated
   * readout error with fp16 layers: 3.5e-4 against 3.2e-4 (profiles/r2_precision_conv_layers.json). */
  const void* conv_w_f16[2];
  /* ---- readout (0 = MER_HUBERT_READOUT_LAST4: the sum of the last four hidden states, as described at
   * mer_hubert_forward) ----
   * MER_HUBERT_READOUT_LAST: hidden_states[-1] alone (MER2023/feature_extraction/audio/extract_transformers_embedding.py,
   * layer_ids = [-1]) into the same out_frames / out_utt: the last layer's output for the post-LN family, the output of
   * encoder.layer_norm after the last layer for the stable-layer-norm family.  Needs n_layers >= 1 (LAST4: >= 4). */
  int readout;
} MerHubertModel;
#define MER_HUBERT_READOUT_LAST4 0
#define MER_HUBERT_READOUT_LAST 1

/* per-row zero-mean / unit-variance (eps 1e-7) of HF Wav2Vec2FeatureExtractor(do_normalize=True)
 * (feature_extraction_wav2vec2.py:78-97), as called at extract_audio_huggingface.py:94.
 * in/out: fp32 [batch, n_samples] with row pitches ld_in / ld_out (floats, each >= n_samples; a shorter pitch is
 * refused).  Mean and variance are taken in double; a row of variance 0 (and any row of one sample) comes out as zeros. */
MER_API int mer_wave_normalize(const float* in, float* out, int batch, int n_samples, long long ld_in,
                               long long ld_out, void* stream);

/* The first layer of the feature encoder on its own: conv0 (Conv1d 1 -> 512, kernel 10, stride 5) of every row of
 * wave (fp32 [batch, n_samples], row pitch ld_wave >= n_samples floats), then
 *   model->feat_norm_layer == 0: GroupNorm(512 groups, eps 1e-5, biased variance over the clip's frames; conv0_w,
 *     gn_g, gn_b) and exact GELU (HF HubertGroupNormConvLayer).  The statistics come from the waveform's tap moments,
 *     summed in double; `frames`: NULL (every clip has T0 = (n_samples - 10) / 5 + 1 frames) or a DEVICE int32 [batch]
 *     of per-clip frame counts in 1 .. T0, over which clip b's statistics are taken (mer_hubert_forward_ragged).
 *   model->feat_norm_layer == 1: + conv_b[0] (NULL: no bias), LayerNorm over the 512 channels (eps 1e-5; conv_ln_g[0],
 *     conv_ln_b[0]) and exact GELU per frame (HF HubertLayerNormConvLayer); `frames` is ignored.
 * out: rows [clip][frame][512] at clip stride out_bstride (elements, >= T0 * 512); out_format MER_EPI_SPLIT_BF16:
 * split-bf16 rows (the BF16X3 operand of conv1), or -- GroupNorm family only, even out_bstride -- MER_EPI_OUT_F16:
 * fp16 rows (the MER_GEMM_F16 operand).  Rows T0 .. of a clip's stride are not written; rows at or past a clip's own
 * frame count are finite and unspecified.  workspace: >= mer_hubert_conv0_workspace_bytes(batch) bytes, 16-byte
 * aligned (GroupNorm statistics; unused by the LayerNorm family).  Refused before any launch: a workspace that is
 * too small or misaligned, a pitch or stride shorter than a row, an output format the family does not write. */
MER_API int mer_hubert_conv0(const MerHubertModel* model, const float* wave, int batch, int n_samples,
                             long long ld_wave, const int* frames, int out_format, void* out, long long out_bstride,
                             void* workspace, long long workspace_bytes, void* stream);
MER_API long long mer_hubert_conv0_workspace_bytes(int batch); /* 5120 * batch */

/* frames produced for n_samples input samples (conv kernels 10,3,3,3,3,2,2 / strides 5,2,2,2,2,2,2) */
MER_API int mer_hubert_num_frames(int n_samples);
MER_API long long mer_hubert_workspace_bytes(int batch, int n_samples);               /* base dims */
MER_API long long mer_hubert_model_workspace_bytes(const MerHubertModel* model, int batch, int n_samples);

/* wave: fp32 [batch, n_samples] raw samples (every row the same length; the reference feeds one
 * clip at a time, or 10 s rows from split_into_batch, extract_audio_huggingface.py:40-50,95).
 * normalize != 0 applies the Wav2Vec2FeatureExtractor zero-mean/unit-variance step per row (:94).
 * Then HubertModel forward (HF modeling_hubert.py) and the readout
 * torch.stack(hidden_states)[[-4,-3,-2,-1]].sum(0) (:98), or hidden_states[-1] (model->readout).
 * Rows of more than 505 frames (clips over 10.1 s) run attention on the fp16 V^T kernel up to MER_ATT_LONG_MAX frames.
 * out_frames: NULL or [batch*T, 768] (FRAME level, :100); out_utt: NULL or [batch, 768] = mean over
 * each row's T frames (UTTERANCE level for clips <= 10 s, :105-108). */
MER_API int mer_hubert_forward(const MerHubertModel* model, const float* wave, int batch, int n_samples,
                               int normalize, void* workspace, long long workspace_bytes,
                               float* out_frames, float* out_utt, float* opt_hidden, void* stream);

/* Ragged batch: row b of wave [batch, n_samples] holds lengths_host[b] <= n_samples samples (HOST array; the rest
 * of the row is ignored when normalize != 0 and must be finite otherwise).  Every clip is computed as if it were
 * forwarded alone, which is what the reference does (one file per model call, extract_audio_huggingface.py:72-100):
 * per-clip waveform normalisation and conv0 GroupNorm statistics, zero padding of the positional conv at the clip's
 * own last frame, attention over the clip's own frames.  T_b = frames of clip b (the conv chain applied to
 * lengths_host[b]).  out_frames: packed [sum_b T_b, hidden] (or NULL); out_utt: [batch, hidden] = mean over the
 * clip's frames.  Needs model->pos_w_bd; workspace as for (batch, n_samples). */
MER_API int mer_hubert_forward_ragged(const MerHubertModel* model, const float* wave, const int* lengths_host,
                                      int batch, int n_samples, int normalize, void* workspace,
                                      long long workspace_bytes, float* out_frames, float* out_utt, void* stream);

/* The part of mer_hubert_forward before the transformer layers: waveform normalisation, the 7-layer conv feature
 * encoder, feature projection, positional convolution (+ encoder.layer_norm for the post-LN family).
 * out_hidden0: [batch * frames, hidden] = hidden_states[0] of the HF model.  Used by the WavLM branch, whose layers
 * (gated relative position bias, HF modeling_wavlm.py WavLMAttention) are orchestrated over the kernel-level entry
 * points below.  Workspace as for mer_hubert_forward. */
MER_API int mer_hubert_frontend(const MerHubertModel* model, const float* wave, int batch, int n_samples, int normalize,
                                void* workspace, long long workspace_bytes, float* out_hidden0, void* stream);

/* ---- WavLM attention pieces (extract_audio_huggingface.py:36-37 wavlm-base / wavlm-large) ------------------- */
/* gate[token, head] = ga * (gb * c[head] - 1) + 2 with (ga, gb) = sigmoid of the two 4-sums of
 * w [8, 64] . x[token, head * 64 : head * 64 + 64] + b [8]   (WavLMAttention.forward steps 1-3). */
MER_API int mer_wavlm_gate(const float* x, long long tokens, int heads, const float* w, const float* b, const float* c,
                           float* gate, void* stream);
/* ctx[b * T + i, h * 64 ...] = softmax_j(q_i . k_j / 8 + rowscale[b * T + i, h] * bias[h, i, j]) v_j over the T tokens
 * of clip b.  qkv: fp32 [batch * T, 3 * heads * 64] (q | k | v); bias: fp32 [heads, T, T]; rowscale: [batch * T, heads]
 * or NULL (= 1).  T <= 1024.  fp32 CUDA-core kernel (not tuned). */
MER_API int mer_biased_attention(const float* qkv, const float* bias, const float* rowscale, int batch, int T, int heads,
                                 float* ctx, int round_tf32_out, void* stream);

/* ---- log mel spectrogram (VGGish front-end) --------------------------------------------------------- */
/* mel_features.log_mel_spectrogram as called by vggish_input.waveform_to_examples
 * (MERBench/feature_extraction/audio/vggish/mel_features.py:166-223, vggish_input.py:66-75,
 * vggish_params.py:22-34): 16 kHz input, 25 ms periodic-Hann frames every 10 ms, |rFFT-512|, 64 HTK mel
 * bands over 125-7500 Hz, log(mel + 0.01).  wave: fp32 [batch, n_samples] (row pitch ld_wave floats);
 * out: fp32 [batch, mer_logmel_num_frames(n_samples), 64]. */
MER_API int mer_logmel_num_frames(int n_samples);
MER_API int mer_logmel(const float* wave, int batch, int n_samples, long long ld_wave, float* out, void* stream);

/* VideoMAE tubelet patches (extract_vision_huggingface.py:147-159; HF VideoMAEPatchEmbeddings): frames uint8 BGR
 * [n_clips * 16, 224, 224, 3] (resized / cropped beforehand) -> out fp32, TF32-rounded [n_clips * 1568, 1536]: the A
 * operand of the patch-embedding GEMM against the flattened Conv3d kernel [hidden, 3 * 2 * 16 * 16]; mean / std are
 * HOST arrays of 3 floats (RGB, the image processor's).  The encoder runs from the host over mer_gemm / mer_layernorm /
 * mer_attention (mertools_b200/extract/videomae.py). */
MER_API int mer_videomae_patchify(const uint8_t* frames_bgr, int n_clips, const float* mean, const float* std,
                                  float* out, void* stream);

/* ---- VideoMAE face-clip encoder of MER2024 / MER2026 (feature_extraction/visual/extract_sun_videomae.py:216-359 over
 * the vendored videomae/modeling_finetune.py VisionTransformer, attn_type 'joint', use_mean_pooling=False). ---- */
typedef struct MerVideoMaeModel {
  int n_layers;          /* 12 (base) / 24 (large) */
  int dim, heads, ffn;   /* 768 / 12 / 3072 or 1024 / 16 / 4096; heads * 64 == dim */
  int img;               /* S: 160 (vit_base_patch16_160) or 224; tokens per view 8 (S / 16)^2 = 800 or 1568 */
  float ln_eps;          /* 1e-6 */
  const void* patch_w;   /* fp16 [dim, 1536]: patch_embed.proj (Conv3d (2, 16, 16)) flattened (c, dt, dy, dx) */
  const float* patch_b;  /* [dim] */
  const float* pos;      /* [tokens per view, dim]: get_sinusoid_encoding_table, fp32 */
  const MerLayerWeights* layers; /* fp16 GEMM weights (MER_GEMM_F16); b_qkv = q_bias | 0 | v_bias */
  const float* norm_g;   /* final norm */
  const float* norm_b;
} MerVideoMaeModel;

/* The tubelet patch operand of n_views clips: frames uint8 [n_frames, S, S, 3] RGB (already resized to S x S; no
 * channel swap, the reference reads them through Image.convert('RGB')), view_rows a DEVICE int32 [n_views, 16] table
 * of frame rows -> out [n_views * 8 (S / 16)^2, 1536], row = (view, tubelet, patch row, patch column), columns in the
 * Conv3d weight's (c, dt, dy, dx) order, value (float(p) / 255 - mean[c]) / std[c] in IEEE fp32 with the ImageNet
 * mean / std (ClipToTensor + Normalize, bit for bit).  out_f32 != 0: fp32; 0: fp16 (round-to-nearest; the patch GEMM's
 * operand).  S is 160 or 224.  A row outside [0, n_frames) is not read: the entries it would feed are NaN. */
MER_API int mer_videomae_clips(const uint8_t* frames, int n_frames, int S, const int32_t* view_rows, int n_views,
                               void* out, int out_f32, void* stream);
/* bytes of workspace for n_views views; -1 for a model mer_videomae_forward refuses (mer_last_error) */
MER_API long long mer_videomae_workspace_bytes(const MerVideoMaeModel* model, int n_views);
/* model(videos, save_feature=True)[1] of the reference (engine_for_finetuning.py:final_test) for n_views views:
 * mer_videomae_clips (fp16), the patch GEMM (+ bias + pos), the pre-LN stack on fp16 operands (erf-GELU, eps ln_eps,
 * the fp16 V^T attention kernel for the 800 / 1568-token rows), the final norm and the mean over each view's tokens.
 * view_rows is a HOST int32 [n_views, 16] table of rows of frames (uint8 [n_frames, img, img, 3] RGB); out: [n_views,
 * dim].  Refused before any launch: a NULL operand, heads * 64 != dim, img other than 160 / 224 (tokens per view
 * outside 254 .. MER_ATT_LONG_MAX), a workspace below mer_videomae_workspace_bytes, a view row outside [0, n_frames). */
MER_API int mer_videomae_forward(const MerVideoMaeModel* model, const uint8_t* frames, int n_frames,
                                 const int32_t* view_rows, int n_views, void* workspace, long long workspace_bytes,
                                 float* out, void* stream);

/* SwiGLU gate of HF Dinov2SwiGLUFFN (dinov2-giant, extract_vision_huggingface.py:135-145): in fp32 [rows, 2 * hidden]
 * = weights_in(x); out [rows, hidden] = silu(in[:, :hidden]) * in[:, hidden:], TF32-rounded when round_tf32_out. */
MER_API int mer_swiglu(const float* in, float* out, long long rows, int hidden, int round_tf32_out, void* stream);

/* ---- LLaMA decoder layers (LlamaModel of the text extractor's LLM branch, extract_text_huggingface.py:170-196): the
 * pieces the GEMM does not cover; the layers are orchestrated from the host over these and mer_gemm
 * (mertools_b200/extract/llama_text.py).  Head dim 128, no grouped-query attention. ---- */
/* SwiGLU of HF LlamaMLP: in fp32 [rows, 2 * hidden] = the fused gate | up GEMM output; out16 fp16 [rows, hidden] =
 * silu(in[:, :hidden]) * in[:, hidden:], the MER_GEMM_F16 operand of down_proj. */
MER_API int mer_swiglu_f16(const float* in, void* out16, long long rows, int hidden, void* stream);
/* HF LlamaRMSNorm over fp32 rows x [rows, dim] (dim % 256 == 0, <= 8192): y = w * (x * rsqrt(mean(x^2) + eps)) with
 * mean(x^2) in fp32.  y16 (optional): fp16 [rows, dim], the operand of the next GEMM.  acc (optional): fp32 [rows, dim]
 * accumulator, acc += y (the final `norm` term of the last-four readout).  At least one of them. */
MER_API int mer_rmsnorm(const float* x, const float* w, void* y16, float* acc, long long rows, int dim, float eps,
                        void* stream);
/* Rotate-half rotary embedding (HF apply_rotary_pos_emb), in place on the q | k columns [0, 2 * heads * 128) of fp16
 * rows qkv16 [tokens, ld]: for every head and j < 64, (x_j, x_j+64) -> (x_j c - x_j+64 s, x_j+64 c + x_j s), c / s =
 * cos_t / sin_t [max_pos, 64] fp32 at the token's position, computed in fp32 and rounded once.  Positions: positions
 * (device int32 [tokens]) when given, else the index inside the packed sequence (cu_seqlens, device [n_seq + 1]).
 * A position outside [0, max_pos) turns the token's q | k into NaN. */
MER_API int mer_rope_f16(void* qkv16, long long ld, long long tokens, int heads, const int32_t* cu_seqlens, int n_seq,
                         const int32_t* positions, const float* cos_t, const float* sin_t, int max_pos, void* stream);
/* mer_rope_f16 over the first rot_heads heads of head_dim 64 or 128 of each row (Falcon: 71 q heads + its one k head),
 * cos_t / sin_t [max_pos, head_dim / 2].  At head_dim 128 with rot_heads = 2 * heads it computes what mer_rope_f16
 * does.  Any other head_dim returns an error before any launch. */
MER_API int mer_rope_hd_f16(void* qkv16, long long ld, long long tokens, int rot_heads, int head_dim,
                            const int32_t* cu_seqlens, int n_seq, const int32_t* positions, const float* cos_t,
                            const float* sin_t, int max_pos, void* stream);
/* Causal softmax(Q K^T / sqrt(128)) V per (sequence, head), head_dim 128 (HF LlamaAttention).  qkv16: fp16 [tokens,
 * 3 * heads * 128] with Q | K column blocks (V columns not read), sequences packed back to back, cu_seqlens [n_seq + 1]
 * (device int32); vt16: fp16 V^T [heads * 128, vt_ld] (vt_ld >= tokens, multiple of 8) as written by mer_gemm's
 * transposed side output; ctx16: fp16 [tokens, heads * 128].  Query i of a sequence attends to its keys 0 .. i; no
 * length cap (max_seqlen sizes the grid).  fp16 P, fp32 softmax statistics: attention_causal.cu. */
MER_API int mer_causal_attention_f16(const void* qkv16, const void* vt16, long long vt_ld, void* ctx16,
                                     const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen, int heads,
                                     void* stream);
/* mer_causal_attention_f16 at head_dim 64, 96 or 128 (HF GPT2Attention: gpt2-chinese-cluecorpussmall at 64,
 * Wenzhong2.0-GPT2-3.5B at 96): qkv16 [tokens, 3 * heads * head_dim], vt16 [heads * head_dim, vt_ld], ctx16 [tokens,
 * heads * head_dim], scores scaled by 1 / sqrt(head_dim).  Any other head_dim returns an error before any launch.  At
 * 128 it runs the same kernel as mer_causal_attention_f16. */
MER_API int mer_causal_attention_hd_f16(const void* qkv16, const void* vt16, long long vt_ld, void* ctx16,
                                        const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen,
                                        int heads, int head_dim, void* stream);

/* ---- pre-LayerNorm decoders with biases (BLOOM / OPT, extract_text_huggingface.py:170-196; orchestrated from the host
 * in mertools_b200/extract/ln_decoder_text.py over these, mer_gemm (MER_EPI_GELU_TANH, MER_EPI_RELU | MER_EPI_OUT_F16)
 * and mer_causal_attention_f16). ---- */
/* mer_causal_attention_f16 with ALiBi (HF BloomAttention): scores q_i . k_j / sqrt(128) + slopes[h] * (j - i) in fp32,
 * i and j counted from the sequence start; HF's slopes[h] * j differs by a per-row constant, which the softmax cancels.
 * slopes: device fp32 [heads] (build_alibi_tensor's).  Same operands and limits otherwise. */
MER_API int mer_causal_alibi_attention_f16(const void* qkv16, const void* vt16, long long vt_ld, void* ctx16,
                                           const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen,
                                           int heads, const float* slopes, void* stream);
/* HF nn.LayerNorm over fp32 rows x [rows, dim] (dim % 256 == 0, <= 8192): y = (x - mean) * rsqrt(var + eps) * gamma +
 * beta, two-pass mean and biased variance in fp32.  Outputs, any non-empty subset: y16 fp16 [rows, dim] (the next GEMM's
 * operand), y32 fp32 [rows, dim] (may not alias x), acc fp32 [rows, dim] with acc += y (the final-norm term of the
 * last-four readout). */
MER_API int mer_layernorm_f16(const float* x, const float* gamma, const float* beta, void* y16, float* y32, float* acc,
                              long long rows, int dim, float eps, void* stream);

/* ---- Falcon-7B (HF FalconModel, parallel attention, multi-query; extract_text_huggingface.py:188-196; orchestrated from
 * the host in mertools_b200/extract/ln_decoder_text.py over these, mer_gemm (MER_EPI_GELU | MER_EPI_OUT_F16) and
 * mer_layernorm_ld_f16, with hidden-wide rows padded to a multiple of 128 columns). ---- */
/* mer_causal_attention_hd_f16 at head_dim 64 with one K / V head shared by every query head (HF FalconAttention,
 * multi_query): qkv16 fp16 [tokens, qkv_ld] with Q in columns [0, heads * 64) and K in [heads * 64, heads * 64 + 64)
 * (other columns not read); vt16 fp16 V^T [64, vt_ld] (vt_ld >= tokens, multiple of 8); ctx16 fp16 [tokens, heads * 64].
 * Scores scaled by 1 / 8; same masking and limits as mer_causal_attention_f16.  Refused with a
 * "mer_causal_mqa_attention_f16:" message before any launch: heads outside 1 .. 65535, qkv_ld below (heads + 1) * 64 or
 * not a multiple of 8, a bad V^T pitch, n_seq outside 1 .. 65535, max_seqlen outside 1 .. tokens, a NULL operand. */
MER_API int mer_causal_mqa_attention_f16(const void* qkv16, long long qkv_ld, const void* vt16, long long vt_ld,
                                         void* ctx16, const int32_t* cu_seqlens, int n_seq, long long tokens,
                                         int max_seqlen, int heads, void* stream);
/* mer_layernorm_f16 over the first dim columns (dim % 64 == 0, <= 8192) of fp32 rows of pitch ld (ld >= dim, multiple
 * of 4); y16 / y32 / acc have the same pitch and only their first dim columns are written.  With ld == dim it computes
 * what mer_layernorm_f16 does. */
MER_API int mer_layernorm_ld_f16(const float* x, long long ld, const float* gamma, const float* beta, void* y16,
                                 float* y32, float* acc, long long rows, int dim, float eps, void* stream);

/* ---- DeBERTa / DeBERTa-v2 encoders (extract_text_huggingface.py:164-166 and the AutoModel branch; orchestrated from the
 * host in mertools_b200/extract/deberta_text.py over this, mer_gemm, mer_layernorm / mer_layernorm_f16 and
 * mer_segment_reduce). ---- */
/* Disentangled self-attention (HF DisentangledSelfAttention, pos_att_type c2p | p2c, head_dim 64) per (sequence, head):
 *   score[i, j] = scale * (q_i . k_j + q_i . pos_k[row] + k_j . pos_q[row]),  row = rel_row[i - j + max_seqlen - 1],
 *   ctx_i = softmax_j(score[i, :]) . V,
 * i and j counted from the sequence start.  qkv, vt, cu_seqlens, tokens, max_seqlen, heads and ctx as mer_attention's
 * V^T form (V columns of qkv not read); pos_k / pos_q: the layer's projections of the relative-position table, [2 span,
 * heads*64] with row pitch pos_ld (elements, >= heads*64, multiple of 8 for fp16 / 4 for fp32), in the operand format
 * of qkv; rel_row: device int32 [2 max_seqlen - 1], values in [0, 2 span) (clamped there).  flags: MER_ATT_QKV_F16 (fp16
 * qkv / vt / tables, m16n8k16) or none (tf32-rounded fp32, m16n8k8), plus at most one of MER_EPI_OUT_F16,
 * MER_EPI_ROUND_TF32, MER_EPI_SPLIT_BF16 for ctx (fp32 otherwise).  qkv, vt, pos_k and pos_q 16-byte aligned.  No
 * length cap.  fp32 scores, softmax statistics and O: attention_rel.cu.  Refused with a "mer_disentangled_attention:"
 * message: heads outside 1 .. 65535, n_seq outside 1 .. 65535, span <= 0, a NULL operand or table, a V^T or table pitch
 * that is too small or misaligned, max_seqlen outside 1 .. tokens, other flags. */
MER_API int mer_disentangled_attention(const void* qkv, const void* vt, long long vt_ld, const void* pos_k,
                                       const void* pos_q, long long pos_ld, int span, const int32_t* rel_row,
                                       float scale, void* ctx, const int32_t* cu_seqlens, int n_seq, long long tokens,
                                       int max_seqlen, int heads, int flags, void* stream);

/* ---- XLNet encoders (xlnet-base-cased, xlnet-large-cased, chinese-xlnet-base: the AutoModel branch of
 * extract_text_huggingface.py; orchestrated from the host in mertools_b200/extract/xlnet_text.py over this, mer_gemm,
 * mer_layernorm and mer_segment_reduce). ---- */
/* XLNet relative self-attention (HF XLNetRelativeAttention.rel_attn_core, attn_type "bi", content stream, head_dim 64)
 * per (sequence, head):
 *   score[i, j] = scale * ((q_i + r_w_bias) . k_j + (q_i + r_r_bias) . r[row] + (q_i + r_s_bias) . seg_embed[s_ij]),
 *   row = rel_row[i - j + max_seqlen - 1],  s_ij = (token_type[i] != token_type[j]),  ctx_i = softmax_j . V,
 * i and j counted from the sequence start.  qkv, vt, cu_seqlens, tokens, max_seqlen, heads and ctx as
 * mer_disentangled_attention (V columns of qkv not read); r: the layer's projection of the relative-position rows,
 * [rows, heads*64] with row pitch r_ld (elements, >= heads*64, multiple of 8 for fp16 / 4 for fp32), in the operand
 * format of qkv; rel_row: device int32 [2 max_seqlen - 1], every value a row of r.  r_w_bias, r_r_bias, r_s_bias:
 * device fp32 [heads, 64]; seg_embed: device fp32 [2, heads, 64]; all four 8-byte aligned.  token_type: device int32
 * [tokens] (absolute token index), or NULL for no segment term (the model called without token_type_ids).  flags as
 * mer_disentangled_attention.  The bias products are fp32 dot products over the operands (q + bias is never rounded to
 * the operand format).  No length cap.  fp32 scores, softmax statistics and O: attention_xl.cu.  Refused with a
 * "mer_xlnet_attention:" message: heads or n_seq outside 1 .. 65535, a NULL operand, table or bias, a V^T or R pitch
 * that is too small or misaligned, a misaligned operand or bias, max_seqlen outside 1 .. tokens, other flags. */
MER_API int mer_xlnet_attention(const void* qkv, const void* vt, long long vt_ld, const void* r, long long r_ld,
                                const int32_t* rel_row, const float* r_w_bias, const float* r_r_bias,
                                const float* r_s_bias, const float* seg_embed, const int32_t* token_type, float scale,
                                void* ctx, const int32_t* cu_seqlens, int n_seq, long long tokens, int max_seqlen,
                                int heads, int flags, void* stream);

/* ---- Whisper branch of the audio extractor (extract_audio_huggingface.py:83-91): the two kernels the shared GEMM /
 * LayerNorm / attention entry points do not cover; the encoder / decoder are orchestrated from the host over those
 * (mertools_b200/extract/whisper.py). ---- */
/* WhisperFeatureExtractor: waves fp32 [batch, ld_wave >= 480000] (30 s at 16 kHz, zero-padded by the caller) ->
 * out fp32 [batch, 3000, ld_out] TIME-MAJOR log-mel features (columns >= 80 zeroed; ld_out = 96 makes it the K-padded
 * operand of the first convolution), TF32-rounded when round_tf32_out.  mel_filters: fp32 [201, 80] (the Slaney bank
 * of the feature extractor).  scratch: int [batch]. */
MER_API int mer_whisper_logmel(const float* waves, int batch, long long ld_wave, const float* mel_filters, float* out,
                               int ld_out, int round_tf32_out, int* scratch, void* stream);
/* softmax(q k^T / 8) v per (clip, head) for nq <= 8 query rows and nk <= 1536 keys (the decoder's causal self-attention
 * over its start tokens, its cross-attention over the encoder frames).  q [batch * nq, ld_q], k / v [batch * nk, ld_*],
 * out [batch * nq, ld_out]; head h uses columns [64 h, 64 h + 64) of each; k rows 16-byte aligned. */
MER_API int mer_small_attention(const float* q, int ld_q, const float* k, int ld_k, const float* v, int ld_v, int batch,
                                int heads, int nq, int nk, int causal, float* out, int ld_out, void* stream);

/* ---- BERT / RoBERTa-base text encoder ------------------------------------------------------------ */
typedef struct MerBertModel {
  int n_layers;
  float ln_eps;             /* 1e-12 (BERT) / 1e-5 (roberta-base checkpoint) */
  const float* word_emb;    /* [V, 768] */
  const float* pos_emb;     /* [P, 768] */
  const float* type_emb0;   /* token_type_embeddings[0], [768] */
  const float* emb_ln_g;
  const float* emb_ln_b;
  const MerLayerWeights* layers;
  /* zero-initialised = the base models; bert-large-uncased / roberta-large / chinese-roberta-wwm-ext-large /
   * chinese-macbert-large ... (extract_text_huggingface.py:21,26,41,49): 1024 / 4096 / 16 */
  int hidden;               /* 0 = 768; 768, 1024 or 256 (embedding tables are then [*, hidden]) */
  int ffn;                  /* 0 = 3072 */
  int heads;                /* 0 = 12; hidden / 64 */
  /* optional: the same layers with fp16 GEMM weights -> the 12 layers run on fp16 operands (one MMA per product
   * instead of three; readout error 2.9e-4 instead of 3.5e-5, profiles/r2_precision_table.json).  NULL: BF16X3. */
  const MerLayerWeights* layers_f16;
} MerBertModel;

MER_API long long mer_bert_workspace_bytes(int tokens, int n_seq); /* base models */
MER_API long long mer_bert_model_workspace_bytes(const MerBertModel* model, int tokens, int n_seq);

/* Packed variable-length batch of tokenised sentences (ids from the HF tokenizer on the host, as in
 * extract_text_huggingface.py:222).  ids/pos_ids: device int32 [tokens]; cu_seqlens: device int32
 * [n_seq+1]; seg_begins/seg_ends: device int32 [n_seq], the token range kept by the reference's
 * outputs[0, start:end] slice (:228-231).  out_tokens: NULL or [tokens, 768] = sum of the last four
 * hidden states (:226); out_utt: NULL or [n_seq, 768] = mean over the kept range (:243-249). */
MER_API int mer_bert_forward(const MerBertModel* model, const int32_t* ids, const int32_t* pos_ids,
                             const int32_t* cu_seqlens, int n_seq, int tokens, int max_seqlen,
                             const int32_t* seg_begins, const int32_t* seg_ends, void* workspace,
                             long long workspace_bytes, float* out_tokens, float* out_utt,
                             float* opt_hidden, void* stream);

/* ELECTRA's factorised embedding (HF ElectraEmbeddings + embeddings_project, modeling_electra.py), for checkpoints whose
 * embedding_size E differs from hidden_size H (ELECTRA-small: E 128, H 256):
 *     e  = LayerNorm_E(word[ids] + pos[pos_ids] + type[0])      (eps: the model's ln_eps)
 *     h0 = e proj_w^T + proj_b                                  (hidden state 0)
 * followed by the model's post-LN layers.  The tables below replace the model's word_emb / pos_emb / type_emb0 /
 * emb_ln_g / emb_ln_b, which are not read.  May only grow at the tail; zero-filled tails = the older behaviour. */
typedef struct MerBertEmbedProjection {
  int emb_dim;              /* E: 128 or 256; 2 E <= the model's ffn (the E-wide rows live in the idle FFN buffer) */
  const float* word_emb;    /* [V, E] */
  const float* pos_emb;     /* [P, E] */
  const float* type_emb0;   /* token_type_embeddings[0], [E] */
  const float* emb_ln_g;    /* [E] */
  const float* emb_ln_b;    /* [E] */
  const float* proj_w;      /* [H, E] as split bf16 rows (read when the model's layers_f16 is NULL: the BF16X3 stack) */
  const void* proj_w_f16;   /* [H, E] fp16 (read when layers_f16 is set: the F16 stack) */
  const float* proj_b;      /* [H] */
} MerBertEmbedProjection;

/* mer_bert_forward with the factorised embedding above (proj != NULL; NULL is exactly mer_bert_forward).  Same
 * arguments, workspace (mer_bert_model_workspace_bytes) and outputs; opt_hidden[0] is the projected h0. */
MER_API int mer_bert_forward_projected(const MerBertModel* model, const MerBertEmbedProjection* proj,
                                       const int32_t* ids, const int32_t* pos_ids, const int32_t* cu_seqlens, int n_seq,
                                       int tokens, int max_seqlen, const int32_t* seg_begins, const int32_t* seg_ends,
                                       void* workspace, long long workspace_bytes, float* out_tokens, float* out_utt,
                                       float* opt_hidden, void* stream);

/* ---- Attention fusion network: forward, loss, backward, Adam ------------------------------------ */
/* toolkit/models/attention.py:8-57 (feat_type 'utt': three MLPEncoders 768->H->H->H, attention MLP
 * 3H->H->H->H, fc_att H->3, weighted sum, heads H->out1 / H->out2), toolkit/utils/loss.py:5-28,
 * main-release.py:50-66,205.  Parameters, gradients and Adam moments are flat fp32 buffers in the
 * reference's state_dict order (audio_encoder.linear_1.weight, .bias, ... fc_out_2.bias). */
typedef struct MerFusionDims {
  int audio_dim, text_dim, video_dim; /* 768 each for the base encoders */
  int hidden;                         /* a multiple of 4, <= 256 */
  int out1;                           /* emotion classes (6), or 0: see below */
  int out2;                           /* valence outputs (1), or 0: see below */
} MerFusionDims;
/* Emotion-only heads (out2 == 0: the MER2024 / MER2025 / MER2026 dataloaders, nn.Linear(hidden, 0) as fc_out_2).
 * Accepted by every fusion entry point, utterance, frame-level and top-N alike.  fc_out_2.weight / .bias are two
 * empty segments at the end of the flat layout (still the state_dict order), the loss is CE alone (loss_out[1] = 0,
 * loss_out[2] = the CE term), and vals, vals_out and d_vals may be NULL -- only when out2 == 0. */
/* Regression-only heads (out1 == 0: the CMU-MOSI / MOSEI, SIMS / SIMSv2 and cross-corpus sentiment dataloaders,
 * nn.Linear(hidden, 0) as fc_out_1).  Accepted by the utterance-level and frame-level entry points when out2 >= 1;
 * the top-N net refuses it, and out1 == out2 == 0 is refused everywhere.  fc_out_1.weight / .bias are two empty
 * segments of the flat layout (between fc_att and fc_out_2), the loss is MSE alone (loss_out[0] = 0, loss_out[2] = the
 * MSE term: emo is never read), and emos, emos_out and d_emos may be NULL -- only when out1 == 0. */

MER_API long long mer_fusion_param_count(const MerFusionDims* dims);
MER_API long long mer_fusion_workspace_bytes(const MerFusionDims* dims, int max_batch);

/* eval-mode forward (no dropout): features [B,hidden], emos_out [B,out1], vals_out [B,out2] —
 * the first three members of the 4-tuple Attention.forward returns (attention.py:52-57). */
MER_API int mer_fusion_forward(const MerFusionDims* dims, const float* params, const float* audios,
                               const float* texts, const float* videos, int batch, void* workspace,
                               long long workspace_bytes, float* features, float* emos_out,
                               float* vals_out, void* stream);

/* train-mode forward + CELoss + MSELoss + backward.  grads receives d(loss)/d(params) with
 * loss = (sum CE + sum SE) * loss_inv_batch (1/batch single-GPU; 1/global_batch under data
 * parallelism so that an all-reduce SUM of grads gives the reference's batch-mean gradient).
 * dropout_p > 0: keep-masks come from a counter hash of (seed, *step_counter, index) unless
 * ext_masks (HOST array of 4 device pointers: audio [B,Da], text, video, concat [B,3H]; entries may
 * be NULL) supplies them (parity tests inject the reference's masks).  The hash index is the element's LOCAL
 * index (row * dim + col of this call's batch), so data-parallel callers must give every rank its own seed:
 * ranks that share one drop the same elements of their local rows, and the all-reduced gradient carries
 * world-size-fold correlated dropout noise (the Python wrappers derive one per rank, fusion.rank_dropout_seed).
 * loss_out: device float[3] = {CE mean, MSE mean, total}. */
MER_API int mer_fusion_fwd_bwd(const MerFusionDims* dims, const float* params, float* grads,
                               const float* audios, const float* texts, const float* videos,
                               const int64_t* emos, const float* vals, int batch, float loss_inv_batch,
                               float dropout_p, unsigned long long seed, const int* step_counter,
                               const float* const* ext_masks, void* workspace, long long workspace_bytes,
                               float* loss_out, float* features, float* emos_out, float* vals_out,
                               void* stream);

/* One whole optimisation step of main-release.py:31-66 (zero_grad, forward, CE + MSE, backward, optional
 * clip_grad_value_, Adam.step) in two launches: a row-parallel cluster kernel (forward, losses, data gradients)
 * and a parameter-parallel kernel in which every weight-gradient element is consumed by its Adam update
 * (torch.optim.Adam(lr, betas, eps, weight_decay) with coupled L2; grad_clip <= 0: no clipping).  Operands as
 * mer_fusion_fwd_bwd; grads still receives the gradient; *step_counter (device int) is read as t-1 and
 * incremented by the kernel.  Data-parallel steps use mer_fusion_fwd_bwd + all-reduce + mer_fusion_adam instead. */
typedef struct MerAdamHyper {
  float lr, beta1, beta2, eps, weight_decay, grad_clip;
} MerAdamHyper;
MER_API int mer_fusion_step(const MerFusionDims* dims, float* params, float* grads, float* exp_avg,
                            float* exp_avg_sq, const float* audios, const float* texts, const float* videos,
                            const int64_t* emos, const float* vals, int batch, float loss_inv_batch,
                            float dropout_p, unsigned long long seed, int* step_counter,
                            const float* const* ext_masks, const MerAdamHyper* adam, void* workspace,
                            long long workspace_bytes, float* loss_out, float* features, float* emos_out,
                            float* vals_out, void* stream);

/* The two halves behind an autograd node (the reference loop calls model(batch), builds the loss itself, then
 * loss.backward(), main-release.py:44-63): train-mode forward (dropout on, masks from (seed, *step_counter) or
 * ext_masks), and the backward pass from the upstream gradients d_features [B,hidden], d_emos [B,out1],
 * d_vals [B,out2] (each may be NULL = zero).  The backward recomputes the forward from the same inputs, seed and
 * step counter (cheaper than keeping activations: 0.48 MMAC per row) and writes d(loss)/d(params) to grads;
 * features / emos_out / vals_out are rewritten as scratch. */
MER_API int mer_fusion_forward_train(const MerFusionDims* dims, const float* params, const float* audios,
                                     const float* texts, const float* videos, int batch, float dropout_p,
                                     unsigned long long seed, const int* step_counter,
                                     const float* const* ext_masks, void* workspace, long long workspace_bytes,
                                     float* features, float* emos_out, float* vals_out, void* stream);
MER_API int mer_fusion_backward(const MerFusionDims* dims, const float* params, float* grads,
                                const float* audios, const float* texts, const float* videos, int batch,
                                const float* d_features, const float* d_emos, const float* d_vals,
                                float dropout_p, unsigned long long seed, const int* step_counter,
                                const float* const* ext_masks, void* workspace, long long workspace_bytes,
                                float* features, float* emos_out, float* vals_out, void* stream);

/* ---- frame-level variant: feat_type = frm_align / frm_unalign (main-release.py:131-142) ----------------
 * Attention with LSTMEncoder per modality (toolkit/models/modules/encoder.py:45-72: nn.LSTM(in, hidden, one
 * layer, batch_first) over the zero-pre-padded sequence -> final hidden state -> dropout -> Linear(hidden,
 * hidden)) in front of the same attention head.  audios / texts / videos are [batch, seq_x, dim_x]; parameters
 * in the reference's state_dict order (rnn.weight_ih_l0, rnn.weight_hh_l0, rnn.bias_ih_l0, rnn.bias_hh_l0,
 * linear_1.weight, linear_1.bias per encoder, then attention_mlp, fc_att, fc_out_1, fc_out_2); hidden is a
 * multiple of 32 up to 128.  Dropout masks 0..2 act on the [batch, hidden] final hidden states.  Everything
 * else as in the utterance-level entry points above. */
MER_API long long mer_fusion_frm_param_count(const MerFusionDims* dims);
MER_API long long mer_fusion_frm_workspace_bytes(const MerFusionDims* dims, int max_batch, int seq_a, int seq_t,
                                                 int seq_v);
MER_API int mer_fusion_frm_forward(const MerFusionDims* dims, const float* params, const float* audios,
                                   const float* texts, const float* videos, int seq_a, int seq_t, int seq_v,
                                   int batch, void* workspace, long long workspace_bytes, float* features,
                                   float* emos_out, float* vals_out, void* stream);
MER_API int mer_fusion_frm_fwd_bwd(const MerFusionDims* dims, const float* params, float* grads,
                                   const float* audios, const float* texts, const float* videos, int seq_a,
                                   int seq_t, int seq_v, const int64_t* emos, const float* vals, int batch,
                                   float loss_inv_batch, float dropout_p, unsigned long long seed,
                                   const int* step_counter, const float* const* ext_masks, void* workspace,
                                   long long workspace_bytes, float* loss_out, float* features, float* emos_out,
                                   float* vals_out, void* stream);

/* ---- Attention_TOPN: N <= 18 utterance-level features (MER2026_Track1/toolkit/models/attention_topn.py) ----
 * One MLPEncoder per feature (encoder0 .. encoder{N-1}), attention_mlp over the N*hidden concat, fc_att
 * [N, hidden], fc_out_1, fc_out_2; parameters in that (state_dict) order.  feats: HOST array of n_feats device
 * pointers.  emos == NULL -> eval-mode forward only.  ext_masks: NULL or HOST array of n_feats + 1 device
 * pointers (per-feature input keep-masks, then the concat mask). */
typedef struct MerFusionTopnDims {
  int n_feats;
  int feat_dims[18];
  int hidden, out1, out2;
} MerFusionTopnDims;
MER_API long long mer_fusion_topn_param_count(const MerFusionTopnDims* dims);
MER_API long long mer_fusion_topn_workspace_bytes(const MerFusionTopnDims* dims, int max_batch);
MER_API int mer_fusion_topn_step(const MerFusionTopnDims* dims, const float* params, float* grads,
                                 const float* const* feats, const int64_t* emos, const float* vals, int batch,
                                 float loss_inv_batch, float dropout_p, unsigned long long seed,
                                 const int* step_counter, const float* const* ext_masks, void* workspace,
                                 long long workspace_bytes, float* loss_out, float* features, float* emos_out,
                                 float* vals_out, void* stream);

/* torch.optim.Adam(lr, betas, eps, weight_decay) with coupled L2, after multiplying the gradient by
 * grad_scale and (grad_clip > 0) clamping it to [-grad_clip, grad_clip] (clip_grad_value_,
 * main-release.py:64-65).  *step_counter (device int) is read as t-1 and incremented. */
MER_API int mer_fusion_adam(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                            long long n, float lr, float beta1, float beta2, float eps,
                            float weight_decay, float grad_scale, float grad_clip, int* step_counter,
                            void* stream);

/* ---- MER2023 baseline nets: MLP and Attention over a free --layers list (MER2023/main-release.py) -------------
 * MLP (:226-245): one chain of Linear -> ReLU -> Dropout per entry of `layers` over the concat A | T | V, then
 * fc_out_1 / fc_out_2 on the chain's output (the features).  Attention (:248-290): such a chain per modality (audio,
 * text, video), attention_mlp (the same chain) over the concat of their outputs, fc_att (layers[last] -> 3, no
 * softmax), the weighted sum of the three outputs (the features), then the two heads.  Parameters, gradients and Adam
 * moments are flat fp32 buffers in state_dict order: module.{0,3,..}.weight/.bias, fc_out_1.*, fc_out_2.* (MLP);
 * audio_mlp.*, text_mlp.*, video_mlp.*, attention_mlp.*, fc_att.*, fc_out_1.*, fc_out_2.* (Attention).
 * Dropout mask t (t = chain * n_layers + layer, chains in the reference's forward order; the MLP has one chain) acts on
 * that layer's [batch, layers[layer]] output.  Limits: 1..8 layers of width 1..1024, input widths 1..65536 (any
 * value: IS10's 1582 and eGeMAPS's 88 included), 1..16 emotion classes, 1..4 valence outputs.  The Attention net
 * refuses a batch of one row: the reference squeezes its [1, L] fused features to a vector and fails. */
#define MER_MLP_KIND_MLP 0
#define MER_MLP_KIND_ATTENTION 1
#define MER_MLP_MAX_LAYERS 8
#define MER_MLP_MAX_WIDTH 1024
#define MER_MLP_MAX_INPUT 65536
#define MER_MLP_MAX_OUT1 16
#define MER_MLP_MAX_OUT2 4
typedef struct MerMlpDims {
  int kind;                            /* MER_MLP_KIND_MLP | MER_MLP_KIND_ATTENTION */
  int audio_dim, text_dim, video_dim;  /* input widths */
  int n_layers;                        /* entries of --layers */
  int layers[MER_MLP_MAX_LAYERS];      /* widths, layers[0 .. n_layers - 1] */
  int out1, out2;                      /* 6 emotion classes, 1 valence */
} MerMlpDims;
/* -1 (mer_last_error says why) for dims or a batch the kernels refuse */
MER_API long long mer_mlp_param_count(const MerMlpDims* dims);
MER_API long long mer_mlp_workspace_bytes(const MerMlpDims* dims, int max_batch);
/* eval-mode forward: features [B, layers[last]], emos_out [B, out1], vals_out [B, out2] */
MER_API int mer_mlp_forward(const MerMlpDims* dims, const float* params, const float* audios, const float* texts,
                            const float* videos, int batch, void* workspace, long long workspace_bytes,
                            float* features, float* emos_out, float* vals_out, void* stream);
/* One training step of main-release.py:334-369: train-mode forward (dropout_p on every layer's output, keep-masks from
 * the counter hash of (seed, *step_counter, mask, element) unless ext_masks -- a HOST array of (1 or 4) * n_layers
 * device keep-masks (0/1), entries may be NULL -- supplies them), CE + MSE averaged over the batch, backward, and with
 * adam != NULL torch.optim.Adam (coupled L2; grad_clip <= 0: none) through mer_fusion_adam, which advances
 * *step_counter.  adam == NULL: grads only, no update, the step counter untouched.  grads receives d(loss)/d(params),
 * loss_out (device float[3]) {CE, MSE, CE + MSE}, features / emos_out / vals_out the train-mode outputs. */
MER_API int mer_mlp_train_step(const MerMlpDims* dims, float* params, float* grads, float* exp_avg,
                               float* exp_avg_sq, const float* audios, const float* texts, const float* videos,
                               const int64_t* emos, const float* vals, int batch, float dropout_p,
                               unsigned long long seed, int* step_counter, const float* const* ext_masks,
                               const MerAdamHyper* adam, void* workspace, long long workspace_bytes,
                               float* loss_out, float* features, float* emos_out, float* vals_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MER_B200_H_ */
