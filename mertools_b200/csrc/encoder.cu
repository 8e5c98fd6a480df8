// encoder.cu — host-side launch sequences of the encoder forwards (no kernels here).
//
// mer_run_stack   : the transformer stack shared by the modalities (dims at run time)
//                   pre-LN  (HF ViTLayer, modeling_vit.py:328-346; CLIPEncoderLayer; the stable-layer-norm
//                            HuBERT encoder) in fp16 / TF32 / BF16X3 operand formats
//                   post-LN (HF HubertEncoderLayer, modeling_hubert.py:372-405; BertLayer) in fp16 / BF16X3
// mer_vit_forward : frames (uint8 BGR) -> patchify -> patch-embed GEMM (+bias +pos) -> stack ->
//                   token-sum readout  (reference: extract_vision_huggingface.py:137-144)
// mer_clip_vision_forward, mer_hubert_forward (base and large families), mer_bert_forward: see each.
//
// Per layer and token the fp16 ViT chain moves: LN 3+1.5 KB x2, QKV 1.5+4.5 KB, attention 4.5+1.5 KB,
// out-proj 1.5+3+3 KB, FC1 1.5+6 KB, FC2 6+3+3 KB = 48 KB (TF32 chain: 72 KB; see DESIGN.md).
#include <vector>

#include "mer_common.cuh"
#include "mer_kernels.h"

constexpr int D = 768;      // base-model dims (ViT-B, HuBERT-base, BERT-base); the large audio family
constexpr int DQKV = 2304;  // passes its own through MerStackArgs / MerHubertModel
constexpr int DFF = 3072;
constexpr int HEADS = 12;

namespace {

int linear(int mode, const float* A, const float* W, const float* bias, const float* res, float* out,
           long long M, int N, int K, int flags, cudaStream_t stream, float* vt = nullptr,
           long long vt_ld = 0, int vt_col0 = 0) {
  MerGemmDesc g;
  memset(&g, 0, sizeof(g));
  g.A = A;
  g.W = W;
  g.rows_per_batch = (int)M;
  g.a_rows_dim = (int)M;
  g.batches = 1;
  g.N = N;
  g.K_inner = K;
  g.taps = 1;
  g.P = 1;
  g.a_phase_stride = K;
  g.a_row_stride = K;
  g.a_batch_stride = (long long)K * M;
  g.ep.bias = bias;
  g.ep.res = res;
  g.ep.out = out;
  g.ep.ld_out = N;
  g.ep.ld_res = N;
  g.ep.flags = flags;
  g.ep.split_off = N;
  g.ep.vt = vt;
  g.ep.vt_ld = vt_ld;
  g.ep.vt_col0 = vt_col0;
  g.mode = mode;
  return mer_gemm_launch(&g, stream);
}

#define MER_TRY(expr)          \
  do {                         \
    if (int _rc = (expr)) return _rc; \
  } while (0)

// mer_attention_launch, except that with `long_rows` (fp16 q | k | V^T rows of 506 .. MER_ATT_LONG_MAX tokens, which
// mer_attention refuses) the call goes to the long-row launch of the same fp16 V^T kernel
int attend(bool long_rows, const float* qkv, const float* vt, long long vt_ld, float* ctx, const int* cu_seqlens,
           int n_seq, long long tokens, int max_seqlen, int heads, int flags, cudaStream_t stream) {
  if (!long_rows)
    return mer_attention_launch(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, max_seqlen, heads, flags, stream);
  const int out_mode = (flags & MER_EPI_OUT_F16) ? 3 : (flags & MER_EPI_SPLIT_BF16) ? 2 : ((flags & MER_EPI_ROUND_TF32) ? 1 : 0);
  return mer_attention_f16_long_launch(qkv, vt, vt_ld, ctx, cu_seqlens, n_seq, tokens, heads, max_seqlen, out_mode,
                                       stream);
}

}  // namespace

int mer_run_stack(const MerStackArgs& a, cudaStream_t stream) {
  MER_REQUIRE(a.tokens > 0 && a.tokens < (1ll << 31), "mer_run_stack: bad token count %lld", a.tokens);
  const long long M = a.tokens;
  // model dims (the file-level constants are the base-model defaults)
  const int D = a.dim > 0 ? a.dim : ::D;
  const int DFF = a.ffn > 0 ? a.ffn : ::DFF;
  const int HEADS = a.heads > 0 ? a.heads : ::HEADS;
  const int DQKV = 3 * D;
  MER_REQUIRE(HEADS * 64 == D, "mer_run_stack: heads %d x 64 != hidden %d", HEADS, D);
  const int ACT = a.quick_gelu ? MER_EPI_QUICK_GELU : MER_EPI_GELU;  // FC1 activation
  const size_t hs_bytes = (size_t)M * D * sizeof(float);
  // EVA02: the rotation needs fp16 q | k, which the pre-LN stacks write exactly when attention takes the fp16 V^T kernel
  const bool rope = a.rope_cos != nullptr;
  if (rope || a.ffn_norms) {
    const bool f16_qk = a.vt && (mer_attention_f16_supported(a.max_seqlen) ||
                                 (a.long_rows && mer_attention_f16_long_supported(a.max_seqlen))) &&
                        (a.mode == MER_GEMM_F16 || !mer_attention_uses_tc(a.max_seqlen));
    MER_REQUIRE(a.pre_ln && (a.mode == MER_GEMM_F16 || a.mode == MER_GEMM_TF32),
                "mer_run_stack: rotary / FFN-norm layers need a pre-LN F16 or TF32 stack");
    MER_REQUIRE(!rope || (a.rope_sin && f16_qk && a.max_seqlen - a.rope_prefix == a.rope_rows &&
                          M % a.max_seqlen == 0),
                "mer_run_stack: rotary table of %d rows for rows of %d tokens (prefix %d) on fp16 q | k", a.rope_rows,
                a.max_seqlen, a.rope_prefix);
    MER_REQUIRE(!a.ffn_norms || DFF <= 3 * D, "mer_run_stack: FFN-norm width %d > 3 x hidden %d", DFF, D);
  }
  if (a.opt_hidden && !a.hidden0_done) MER_CUDA_CHECK(cudaMemcpyAsync(a.opt_hidden, a.x, hs_bytes, cudaMemcpyDeviceToDevice, stream));
  for (int l = 0; l < a.n_layers; ++l) {
    const MerLayerWeights& w = a.layers[l];
    const int first_acc = a.n_layers - a.acc_last;  // hidden state index l+1 > first_acc is summed
    // operand format of the tensor-core inputs in this stack: tf32-rounded fp32, or split bf16
    const bool split = a.mode == MER_GEMM_BF16X3;
    // V^T attention (sequences <= 253): the QKV GEMM writes V transposed into a.vt instead of
    // the V columns of qkv
    // (254 .. 505 tokens, and up to MER_ATT_LONG_MAX with a.long_rows: the fp16 V^T kernel, which takes fp16
    // q | k | V^T whatever the stack's operand format)
    const bool f16_long = a.long_rows && a.vt && mer_attention_f16_long_supported(a.max_seqlen);
    const bool f16_rows = f16_long || mer_attention_f16_supported(a.max_seqlen);
    const bool long_att = a.vt && !mer_attention_uses_tc(a.max_seqlen) && f16_rows;
    float* vt = (a.vt && (long_att || mer_attention_uses_tc(a.max_seqlen))) ? a.vt : nullptr;
    // the TF32 / BF16X3 stacks: QKV epilogue and attention flags (q | k | v tf32-rounded fp32, or fp16 = the same 10-bit
    // mantissa, for the long-key kernel)
    const int qkv_fl = long_att ? MER_EPI_OUT_F16 : MER_EPI_ROUND_TF32;
    const int att_in = long_att ? MER_ATT_QKV_F16 : 0;
    const int opnd = split ? MER_EPI_SPLIT_BF16 : MER_EPI_ROUND_TF32;
    if (a.pre_ln && a.mode == MER_GEMM_F16) {
      // same chain on fp16 operands: LN, the QKV GEMM (q | k rows and V^T), attention and FC1 write fp16
      // into the (fp32-sized) scratch buffers; only the residual stream x stays fp32
      float* xn16 = a.xn;  // fp16 [M, 768]
      float* h16 = a.h;    // fp16 [M, 3072]
      const bool f16_att = vt != nullptr && f16_rows;
      MER_TRY(mer_layernorm_launch(a.x, w.ln1_g, w.ln1_b, xn16, nullptr, nullptr, M, D, a.eps, MER_LN_OUT_F16,
                                   stream));
      if (f16_att) {
        MER_TRY(linear(a.mode, xn16, w.w_qkv, w.b_qkv, nullptr, a.qkv, M, DQKV, D, MER_EPI_OUT_F16, stream,
                       vt, a.vt_ld, 2 * D));
        if (rope)
          MER_TRY(mer_rope2d_f16(a.qkv, DQKV, M, a.max_seqlen, a.rope_prefix, HEADS, 64, a.rope_cos, a.rope_sin,
                                 a.rope_rows, stream));
        MER_TRY(attend(f16_long, a.qkv, vt, a.vt_ld, xn16, a.cu_seqlens, a.n_seq, M, a.max_seqlen, HEADS,
                       MER_EPI_OUT_F16 | MER_ATT_QKV_F16, stream));
        MER_TRY(linear(a.mode, xn16, w.w_o, w.b_o, a.x, a.x, M, D, D, 0, stream));
      } else {
        // sequences beyond the fp16 attention kernels (> 505 tokens: a CLIP tower forced to fp16 at a larger image;
        // no caller at image 224 reaches this): the linear layers stay on fp16
        // operands, attention runs the fp32-operand flash kernel on a TF32-rounded fp32 q | k | v (same 10-bit
        // mantissa) and its fp32 context is cast to the fp16 out-proj operand through the idle FFN buffer
        MER_TRY(linear(a.mode, xn16, w.w_qkv, w.b_qkv, nullptr, a.qkv, M, DQKV, D, MER_EPI_ROUND_TF32, stream));
        MER_TRY(mer_attention_launch(a.qkv, nullptr, 0, a.xn, a.cu_seqlens, a.n_seq, M, a.max_seqlen, HEADS, 0, stream));
        MER_TRY(mer_cast_f16_launch(a.xn, h16, M * D, stream));
        MER_TRY(linear(a.mode, h16, w.w_o, w.b_o, a.x, a.x, M, D, D, 0, stream));
      }
      MER_TRY(mer_layernorm_launch(a.x, w.ln2_g, w.ln2_b, xn16, nullptr, nullptr, M, D, a.eps, MER_LN_OUT_F16,
                                   stream));
      if (a.ffn_norms) {  // EVA02: x += fc2(LN(silu(fc1_g h) * fc1_x h)), the normed product in the dead qkv buffer
        MER_TRY(linear(a.mode, xn16, w.w_fc1, w.b_fc1, nullptr, a.h, M, 2 * DFF, D, 0, stream));
        MER_TRY(mer_swiglu_ln(a.h, a.ffn_norms[l].g, a.ffn_norms[l].b, a.eps, a.qkv, M, DFF, 1, stream));
        MER_TRY(linear(a.mode, a.qkv, w.w_fc2, w.b_fc2, a.x, a.x, M, D, DFF, 0, stream));
      } else {
        MER_TRY(linear(a.mode, xn16, w.w_fc1, w.b_fc1, nullptr, h16, M, DFF, D, ACT | MER_EPI_OUT_F16,
                       stream));
        MER_TRY(linear(a.mode, h16, w.w_fc2, w.b_fc2, a.x, a.x, M, D, DFF, 0, stream));
      }
    } else if (a.pre_ln) {
      // x = x + Wo * Attn(LN1(x));  x = x + W2 * GELU(W1 * LN2(x))
      MER_TRY(mer_layernorm_launch(a.x, w.ln1_g, w.ln1_b, split ? nullptr : a.xn, split ? a.xn : nullptr,
                                   nullptr, M, D, a.eps, MER_LN_ROUND_TF32, stream));
      MER_TRY(linear(a.mode, a.xn, w.w_qkv, w.b_qkv, nullptr, a.qkv, M, DQKV, D, qkv_fl, stream,
                     vt, a.vt_ld, 2 * D));
      if (rope)
        MER_TRY(mer_rope2d_f16(a.qkv, DQKV, M, a.max_seqlen, a.rope_prefix, HEADS, 64, a.rope_cos, a.rope_sin,
                               a.rope_rows, stream));
      MER_TRY(attend(f16_long, a.qkv, vt, a.vt_ld, a.xn, a.cu_seqlens, a.n_seq, M, a.max_seqlen, HEADS,
                     opnd | att_in, stream));
      MER_TRY(linear(a.mode, a.xn, w.w_o, w.b_o, a.x, a.x, M, D, D, 0, stream));
      MER_TRY(mer_layernorm_launch(a.x, w.ln2_g, w.ln2_b, split ? nullptr : a.xn, split ? a.xn : nullptr,
                                   nullptr, M, D, a.eps, MER_LN_ROUND_TF32, stream));
      if (a.ffn_norms) {  // EVA02 (TF32 stack): the normed product tf32-rounded in the dead qkv buffer
        MER_TRY(linear(a.mode, a.xn, w.w_fc1, w.b_fc1, nullptr, a.h, M, 2 * DFF, D, 0, stream));
        MER_TRY(mer_swiglu_ln(a.h, a.ffn_norms[l].g, a.ffn_norms[l].b, a.eps, a.qkv, M, DFF, 0, stream));
        MER_TRY(linear(a.mode, a.qkv, w.w_fc2, w.b_fc2, a.x, a.x, M, D, DFF, 0, stream));
      } else {
        MER_TRY(linear(a.mode, a.xn, w.w_fc1, w.b_fc1, nullptr, a.h, M, DFF, D, ACT | opnd, stream));
        MER_TRY(linear(a.mode, a.h, w.w_fc2, w.b_fc2, a.x, a.x, M, D, DFF, 0, stream));
      }
    } else if (a.mode == MER_GEMM_F16) {
      // post-LN on fp16 operands (scripts/precision_table.py): x stays the exact fp32 LayerNorm output
      // (residual stream, hidden state), xs carries its fp16 copy (GEMM operand, written by the same LayerNorm
      // pass); ctx and the FC1 output are fp16; the pre-LN sums are fp32.
      float* x16 = a.xs;
      float* c16 = a.xn;   // fp16 ctx; later the fp32 pre-LN sum of the FFN half
      float* h16 = a.h;
      const bool f16_att = vt != nullptr && f16_rows;
      if (f16_att) {
        MER_TRY(linear(a.mode, x16, w.w_qkv, w.b_qkv, nullptr, a.qkv, M, DQKV, D, MER_EPI_OUT_F16, stream, vt,
                       a.vt_ld, 2 * D));
        MER_TRY(attend(f16_long, a.qkv, vt, a.vt_ld, c16, a.cu_seqlens, a.n_seq, M, a.max_seqlen, HEADS,
                       MER_EPI_OUT_F16 | MER_ATT_QKV_F16, stream));
        MER_TRY(linear(a.mode, c16, w.w_o, w.b_o, a.x, a.qkv, M, D, D, 0, stream));  // qkv is dead: holds the sum
      } else {
        // rows beyond the fp16 attention kernels (> MER_ATT_LONG_MAX frames with long_rows, > 505 tokens without):
        // TF32-rounded fp32 q | k | v (same 10-bit mantissa)
        // through the fp32-operand attention kernels, fp32 context cast to the fp16 out-proj operand
        MER_TRY(linear(a.mode, x16, w.w_qkv, w.b_qkv, nullptr, a.qkv, M, DQKV, D, MER_EPI_ROUND_TF32, stream, vt,
                       a.vt_ld, 2 * D));
        MER_TRY(mer_attention_launch(a.qkv, vt, a.vt_ld, a.xn, a.cu_seqlens, a.n_seq, M, a.max_seqlen, HEADS, 0,
                                     stream));
        MER_TRY(mer_cast_f16_launch(a.xn, h16, M * D, stream));
        MER_TRY(linear(a.mode, h16, w.w_o, w.b_o, a.x, a.qkv, M, D, D, 0, stream));
      }
      MER_TRY(mer_layernorm_launch(a.qkv, w.ln1_g, w.ln1_b, a.x, x16, nullptr, M, D, a.eps, MER_LN_SPLIT_F16, stream));
      MER_TRY(linear(a.mode, x16, w.w_fc1, w.b_fc1, nullptr, h16, M, DFF, D, MER_EPI_GELU | MER_EPI_OUT_F16, stream));
      MER_TRY(linear(a.mode, h16, w.w_fc2, w.b_fc2, a.x, a.xn, M, D, DFF, 0, stream));
      int fl = MER_LN_SPLIT_F16;
      float* acc = nullptr;
      if (a.acc && a.acc_last > 0 && l + 1 > first_acc) {
        acc = a.acc;
        fl |= (l + 1 == first_acc + 1) ? MER_LN_ACC_INIT : MER_LN_ACC_ADD;
      }
      MER_TRY(mer_layernorm_launch(a.xn, w.ln2_g, w.ln2_b, a.x, x16, acc, M, D, a.eps, fl, stream));
    } else {
      // x = LN1(x + Wo * Attn(x));  x = LN2(x + W2 * GELU(W1 * x)).
      // TF32: x itself is tf32-rounded and doubles as the GEMM operand.  BF16X3: x stays exact fp32
      // (residual) and xs carries its split copy (GEMM operand).
      const float* xop = split ? a.xs : a.x;
      MER_TRY(linear(a.mode, xop, w.w_qkv, w.b_qkv, nullptr, a.qkv, M, DQKV, D, qkv_fl, stream,
                     vt, a.vt_ld, 2 * D));
      MER_TRY(attend(f16_long, a.qkv, vt, a.vt_ld, a.xn, a.cu_seqlens, a.n_seq, M, a.max_seqlen, HEADS,
                     opnd | att_in, stream));
      // the pre-LN sum goes to the (now dead) qkv buffer: ctx in xn is still being read
      MER_TRY(linear(a.mode, a.xn, w.w_o, w.b_o, a.x, a.qkv, M, D, D, 0, stream));
      MER_TRY(mer_layernorm_launch(a.qkv, w.ln1_g, w.ln1_b, a.x, split ? a.xs : nullptr, nullptr, M, D,
                                   a.eps, split ? 0 : MER_LN_ROUND_TF32, stream));
      MER_TRY(linear(a.mode, xop, w.w_fc1, w.b_fc1, nullptr, a.h, M, DFF, D, MER_EPI_GELU | opnd, stream));
      MER_TRY(linear(a.mode, a.h, w.w_fc2, w.b_fc2, a.x, a.xn, M, D, DFF, 0, stream));
      int fl = split ? 0 : MER_LN_ROUND_TF32;
      float* acc = nullptr;
      if (a.acc && a.acc_last > 0 && l + 1 > first_acc) {
        acc = a.acc;
        fl |= (l + 1 == first_acc + 1) ? MER_LN_ACC_INIT : MER_LN_ACC_ADD;
      }
      MER_TRY(mer_layernorm_launch(a.xn, w.ln2_g, w.ln2_b, a.x, split ? a.xs : nullptr, acc, M, D, a.eps,
                                   fl, stream));
    }
    if (a.opt_hidden) {
      // post-LN: the hidden state is the un-rounded LayerNorm output; re-derive it exactly from
      // the pre-LN sum still sitting in xn (debug/parity path only)
      float* dst = a.opt_hidden + (size_t)(l + 1) * M * D;
      if (a.pre_ln) {
        MER_CUDA_CHECK(cudaMemcpyAsync(dst, a.x, hs_bytes, cudaMemcpyDeviceToDevice, stream));
      } else {
        MER_TRY(mer_layernorm_launch(a.xn, w.ln2_g, w.ln2_b, dst, nullptr, nullptr, M, D, a.eps, 0, stream));
      }
    }
  }
  return 0;
}

extern "C" {

long long mer_vit_workspace_bytes(int n_frames) {
  const long long M = (long long)n_frames * 197;
  // x, xn, qkv, h (+ patch operand aliasing h), V^T + offsets
  return (M * (D + D + DQKV + DFF) + (long long)D * ((M + 7) & ~7ll)) * 4 + ((long long)n_frames + 1) * 4 + 1024;
}

int mer_vit_forward(const MerVitModel* m, const uint8_t* frames_bgr, int n_frames, void* workspace,
                    long long workspace_bytes, float* out_frame_feats, float* opt_hidden,
                    void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(m && frames_bgr && workspace && out_frame_feats, "mer_vit_forward: null operand");
  MER_REQUIRE(n_frames > 0, "mer_vit_forward: n_frames=%d", n_frames);
  MER_REQUIRE(workspace_bytes >= mer_vit_workspace_bytes(n_frames),
              "mer_vit_forward: workspace %lld B < required %lld B", workspace_bytes,
              mer_vit_workspace_bytes(n_frames));
  MER_REQUIRE((long long)n_frames * 197 < (1ll << 31) / 4, "mer_vit_forward: too many frames");
  const long long M = (long long)n_frames * 197;
  float* x = static_cast<float*>(workspace);
  float* xn = x + M * D;
  float* qkv = xn + M * D;
  float* h = qkv + M * DQKV;
  float* vt = h + M * DFF;
  const long long vt_ld = (M + 7) & ~7ll;  // fp32 or fp16 V^T rows start on 16-byte boundaries
  int* offsets = reinterpret_cast<int*>(vt + (long long)D * vt_ld);
  float* a_patch = h;  // [n_frames*196, 768] patch operand lives in the (not yet used) FFN buffer

  MER_TRY(mer_iota_offsets_launch(offsets, n_frames, 197, stream));
  MER_TRY(mer_vit_patchify_launch(frames_bgr, n_frames, a_patch, stream));
  MER_TRY(mer_vit_cls_rows_launch(m->cls_pos0, x, n_frames, stream));
  {
    MerGemmDesc g;
    memset(&g, 0, sizeof(g));
    g.A = a_patch;
    g.W = m->patch_w;
    g.rows_per_batch = 196;
    g.a_rows_dim = 196;
    g.batches = n_frames;
    g.N = D;
    g.K_inner = D;
    g.taps = 1;
    g.P = 1;
    g.a_phase_stride = D;
    g.a_row_stride = D;
    g.a_batch_stride = 196ll * D;
    g.ep.bias = m->patch_b;
    g.ep.res = m->pos_rest;  // + position_embeddings[1:], same for every frame
    g.ep.res_bstride = 0;
    g.ep.out = x;
    g.ep.out_bstride = 197;
    g.ep.out_row0 = 1;
    g.ep.ld_out = D;
    g.ep.ld_res = D;
    g.mode = MER_GEMM_TF32;
    MER_TRY(mer_gemm_launch(&g, stream));
  }
  MerStackArgs a;
  memset(&a, 0, sizeof(a));
  a.layers = m->layers;
  a.n_layers = m->n_layers;
  a.pre_ln = 1;
  MER_REQUIRE(m->gemm_mode == MER_GEMM_TF32 || m->gemm_mode == MER_GEMM_F16,
              "mer_vit_forward: gemm_mode %d (MER_GEMM_TF32 or MER_GEMM_F16)", m->gemm_mode);
  a.mode = m->gemm_mode;
  a.eps = m->ln_eps;
  a.tokens = M;
  a.cu_seqlens = offsets;
  a.n_seq = n_frames;
  a.max_seqlen = 197;
  a.x = x;
  a.xn = xn;
  a.qkv = qkv;
  a.h = h;
  a.vt = vt;
  a.vt_ld = vt_ld;
  a.opt_hidden = opt_hidden;
  MER_TRY(mer_run_stack(a, stream));
  MER_TRY(mer_segment_reduce_launch(x, offsets, offsets + 1, n_frames, D, MER_SEG_SUM, out_frame_feats, stream));
  return 0;
}

// ------------------------------------------------------------------------------------------------
// CLIP vision tower
// ------------------------------------------------------------------------------------------------
struct ClipPlan { long long M, vt_ld, off_x, off_xn, off_qkv, off_h, off_vt, off_cu, total; int tokens, P; };

static ClipPlan clip_plan(const MerClipVisionModel* m, int n_frames) {
  ClipPlan p;
  const int g = m->image / m->patch;
  p.P = g * g;
  p.tokens = p.P + 1;
  p.M = (long long)n_frames * p.tokens;
  p.vt_ld = (p.M + 7) & ~7ll;
  auto al = [](long long x) { return (x + 255) & ~255ll; };
  const long long D = m->hidden;
  long long o = 0;
  p.off_x = o;   o += al(p.M * D * 4);
  p.off_xn = o;  o += al(p.M * D * 4);
  p.off_qkv = o; o += al(p.M * 3 * D * 4);
  // EVA02's FC1 writes the gate and value halves side by side: 2 ffn fp32 columns
  const long long hcols = m->variant == MER_VISION_EVA02 ? 2ll * m->ffn : m->ffn;
  long long hb = p.M * hcols * 4, pb = (long long)n_frames * p.P * m->kpad * 4;
  p.off_h = o;   o += al(hb > pb ? hb : pb);   // FFN buffer; the patch operand lives here first
  p.off_vt = o;  o += al(D * p.vt_ld * 4);
  p.off_cu = o;  o += al(((long long)n_frames + 1) * 4);
  p.total = o;
  return p;
}

long long mer_clip_vision_workspace_bytes(const MerClipVisionModel* m, int n_frames) {
  if (!m || m->patch <= 0 || m->image % m->patch) return -1;
  return clip_plan(m, n_frames).total;
}

int mer_clip_vision_forward(const MerClipVisionModel* m, const uint8_t* frames_bgr, int n_frames, int H, int W,
                            int crop_y0, int crop_x0, void* workspace, long long workspace_bytes,
                            float* out_embeds, float* opt_hidden, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(m && frames_bgr && workspace && out_embeds && n_frames > 0, "mer_clip_vision_forward: bad operands");
  const int D = m->hidden;
  MER_REQUIRE((D == 768 || D == 1024 || (D == 1536 && m->variant == MER_VISION_EMBED_ONLY)) && m->heads * 64 == D &&
                  m->ffn % 128 == 0 && m->proj_dim % 128 == 0 &&
                  m->image % m->patch == 0 && m->kpad % 32 == 0 && m->kpad >= 3 * m->patch * m->patch,
              "mer_clip_vision_forward: unsupported dims (hidden %d, heads %d, ffn %d, proj %d, patch %d)", D,
              m->heads, m->ffn, m->proj_dim, m->patch);
  MER_REQUIRE(m->gemm_mode == MER_GEMM_TF32 || m->gemm_mode == MER_GEMM_F16, "mer_clip_vision_forward: gemm_mode");
  const ClipPlan p = clip_plan(m, n_frames);
  MER_REQUIRE(workspace_bytes >= p.total, "mer_clip_vision_forward: workspace %lld B < required %lld B",
              workspace_bytes, p.total);
  MER_REQUIRE(p.M < (1ll << 31) / 4, "mer_clip_vision_forward: too many frames");
  const bool dinov2 = m->variant == MER_VISION_DINOV2, eva02 = m->variant == MER_VISION_EVA02;
  MER_REQUIRE(m->variant >= MER_VISION_CLIP && m->variant <= MER_VISION_EVA02, "mer_clip_vision_forward: variant %d",
              m->variant);
  MER_REQUIRE(m->variant != MER_VISION_CLIP ? (m->pre_ln_g == nullptr && m->proj_dim == D)
                                            : (m->pre_ln_g && m->post_ln_g && m->proj_w),
              "mer_clip_vision_forward: variant %d operands", m->variant);
  if (eva02) {
    MER_REQUIRE(m->rope_cos && m->rope_sin && m->ffn_norms && m->post_ln_g && m->post_ln_b,
                "mer_clip_vision_forward: EVA02 needs rope tables, FFN norms and fc_norm");
    MER_REQUIRE(m->rope_rows == p.P, "mer_clip_vision_forward: EVA02 rope table of %d rows for %d patches",
                m->rope_rows, p.P);
    MER_REQUIRE(m->ffn <= 3 * D && m->ffn <= 4096, "mer_clip_vision_forward: EVA02 FFN width %d (up to min(3 x %d, 4096))",
                m->ffn, D);
    MER_REQUIRE(mer_attention_f16_supported(p.tokens),
                "mer_clip_vision_forward: EVA02 needs the fp16 attention rows (%d tokens)", p.tokens);
    for (int l = 0; l < m->n_layers; ++l)
      MER_REQUIRE(m->ffn_norms[l].g && m->ffn_norms[l].b, "mer_clip_vision_forward: EVA02 FFN norm %d is NULL", l);
  }
  char* ws = static_cast<char*>(workspace);
  float* x = reinterpret_cast<float*>(ws + p.off_x);
  float* xn = reinterpret_cast<float*>(ws + p.off_xn);
  float* qkv = reinterpret_cast<float*>(ws + p.off_qkv);
  float* h = reinterpret_cast<float*>(ws + p.off_h);
  float* vt = reinterpret_cast<float*>(ws + p.off_vt);
  int* offsets = reinterpret_cast<int*>(ws + p.off_cu);
  float* a_patch = h;
  MER_TRY(mer_iota_offsets_launch(offsets, n_frames, p.tokens, stream));
  MER_TRY(mer_patchify_generic_launch(frames_bgr, n_frames, H, W, crop_y0, crop_x0, m->image, m->patch, m->kpad,
                                      m->mean, m->std, a_patch, stream));
  MER_TRY(mer_cls_rows_generic_launch(m->cls_pos0, x, n_frames, p.tokens, D, stream));
  {
    MerGemmDesc g;
    memset(&g, 0, sizeof(g));
    g.A = a_patch;
    g.W = m->patch_w;
    g.rows_per_batch = p.P;
    g.a_rows_dim = p.P;
    g.batches = n_frames;
    g.N = D;
    g.K_inner = m->kpad;
    g.taps = 1;
    g.P = 1;
    g.a_phase_stride = m->kpad;
    g.a_row_stride = m->kpad;
    g.a_batch_stride = (long long)p.P * m->kpad;
    g.ep.res = m->pos_rest;  // + position_embedding[1:], same for every frame (no conv bias in CLIP)
    g.ep.res_bstride = 0;
    g.ep.out = x;
    g.ep.out_bstride = p.tokens;
    g.ep.out_row0 = 1;
    g.ep.ld_out = D;
    g.ep.ld_res = D;
    g.mode = MER_GEMM_TF32;
    MER_TRY(mer_gemm_launch(&g, stream));
  }
  if (m->variant == MER_VISION_EMBED_ONLY) {  // the embedding output (hidden_states[0]) for a host-orchestrated stack
    MER_CUDA_CHECK(cudaMemcpyAsync(out_embeds, x, (size_t)p.M * D * 4, cudaMemcpyDeviceToDevice, stream));
    return 0;
  }
  if (m->variant == MER_VISION_CLIP)
    MER_TRY(mer_layernorm_launch(x, m->pre_ln_g, m->pre_ln_b, x, nullptr, nullptr, p.M, D, m->ln_eps, 0, stream));
  MerStackArgs a;
  memset(&a, 0, sizeof(a));
  a.layers = m->layers;
  a.n_layers = m->n_layers;
  a.pre_ln = 1;
  a.mode = m->gemm_mode;
  a.dim = D;
  a.ffn = m->ffn;
  a.heads = m->heads;
  a.quick_gelu = dinov2 ? 0 : 1;
  a.eps = m->ln_eps;
  a.tokens = p.M;
  a.cu_seqlens = offsets;
  a.n_seq = n_frames;
  a.max_seqlen = p.tokens;
  a.x = x;
  a.xn = xn;
  a.qkv = qkv;
  a.h = h;
  a.vt = vt;
  a.vt_ld = p.vt_ld;
  a.opt_hidden = opt_hidden;
  if (eva02) {
    a.rope_cos = m->rope_cos;
    a.rope_sin = m->rope_sin;
    a.rope_rows = m->rope_rows;
    a.rope_prefix = 1;
    a.ffn_norms = m->ffn_norms;
  }
  MER_TRY(mer_run_stack(a, stream));
  if (dinov2)  // hidden_states[-1].sum(dim=1): every token of the last layer's output, per frame
    return mer_segment_reduce_launch(x, offsets, offsets + 1, n_frames, D, MER_SEG_SUM, out_embeds, stream);
  if (eva02) {  // timm forward_head, global_pool 'avg': mean over the patch rows, then fc_norm
    int* begins = reinterpret_cast<int*>(qkv);  // the QKV buffer is dead now
    int* ends = begins + n_frames;
    float* pooled = reinterpret_cast<float*>(ws + p.off_vt);
    MER_TRY(mer_frame_spans_launch(begins, ends, n_frames, p.tokens, 1, stream));
    MER_TRY(mer_segment_reduce_launch(x, begins, ends, n_frames, D, MER_SEG_MEAN, pooled, stream));
    return mer_layernorm_launch(pooled, m->post_ln_g, m->post_ln_b, out_embeds, nullptr, nullptr, n_frames, D,
                                m->ln_eps, 0, stream);
  }
  // class-token rows -> post_layernorm (tf32-rounded: GEMM operand) -> visual_projection
  float* cls = qkv;                        // [n_frames, D]   (the QKV buffer is dead now)
  float* pooled = qkv + (long long)n_frames * D;
  MER_TRY(mer_gather_rows_launch(x, 0, p.tokens, n_frames, D, cls, stream));
  MER_TRY(mer_layernorm_launch(cls, m->post_ln_g, m->post_ln_b, pooled, nullptr, nullptr, n_frames, D, m->ln_eps,
                               MER_LN_ROUND_TF32, stream));
  MER_TRY(linear(MER_GEMM_TF32, pooled, m->proj_w, nullptr, nullptr, out_embeds, n_frames, m->proj_dim, D, 0, stream));
  return 0;
}

// ------------------------------------------------------------------------------------------------
// HuBERT
// ------------------------------------------------------------------------------------------------
static const int kHubK[7] = {10, 3, 3, 3, 3, 2, 2};
static const int kHubS[7] = {5, 2, 2, 2, 2, 2, 2};

struct HubertPlan {
  int T[7];      // frames after conv i
  int Tpad[7];   // allocated rows per clip (even)
  long long off_wave, off_stats, off_ping, off_pong, off_x, off_xs, off_xn, off_qkv, off_h, off_acc,
      off_vt, off_cu, off_meta, total;
  long long M;
};

static HubertPlan hubert_plan(int B, int L, int D = ::D, int DFF = ::DFF) {
  const int DQKV = 3 * D;
  HubertPlan p;
  int t = L;
  for (int i = 0; i < 7; ++i) {
    t = (t - kHubK[i]) / kHubS[i] + 1;
    if (t < 0) t = 0;
    p.T[i] = t;
    p.Tpad[i] = (t + 1) & ~1;
  }
  p.M = (long long)B * p.T[6];
  auto al = [](long long x) { return (x + 255) & ~255ll; };
  long long o = 0;
  p.off_wave = o;  o += al((long long)B * L * 4);
  p.off_stats = o; o += al((long long)B * 512 * 2 * 8);
  p.off_ping = o;  o += al((long long)B * p.Tpad[0] * 512 * 4);
  p.off_pong = o;  o += al((long long)B * p.Tpad[1] * 512 * 4);
  p.off_x = o;     o += al(p.M * D * 4);
  p.off_xs = o;    o += al(p.M * D * 4);
  p.off_xn = o;    o += al(p.M * D * 4);
  p.off_qkv = o;   o += al(p.M * DQKV * 4);
  p.off_h = o;     o += al(p.M * DFF * 4);
  p.off_acc = o;   o += al(p.M * D * 4);
  p.off_vt = o;    o += al((long long)D * ((p.M + 7) & ~7ll) * 4);
  p.off_cu = o;    o += al(((long long)B + 1) * 4);
  p.off_meta = o;  o += al((4ll * B + 4) * 4);  // ragged batches: samples, conv0 frames, frames, cu_seqlens per clip
  p.total = o;
  return p;
}

static int hub_dim(const MerHubertModel* m) { return m->hidden > 0 ? m->hidden : ::D; }
static int hub_ffn(const MerHubertModel* m) { return m->ffn > 0 ? m->ffn : ::DFF; }
static int hub_heads(const MerHubertModel* m) { return m->heads > 0 ? m->heads : ::HEADS; }

long long mer_hubert_model_workspace_bytes(const MerHubertModel* m, int batch, int n_samples) {
  if (!m) return -1;
  return hubert_plan(batch, n_samples, hub_dim(m), hub_ffn(m)).total;
}

int mer_hubert_num_frames(int n_samples) { return hubert_plan(1, n_samples).T[6]; }

long long mer_hubert_workspace_bytes(int batch, int n_samples) {
  return hubert_plan(batch, n_samples).total;
}

// lengths_host == nullptr: B equal-length rows of L samples.  Otherwise a RAGGED batch: row b holds
// lengths_host[b] <= L samples (the rest of the row is ignored), every clip is computed as if it ran alone
// (the reference feeds one file at a time, extract_audio_huggingface.py:72-100): waveform normalisation and the
// GroupNorm statistics of conv0 use the clip's own extent, conv1..6 / projection run on the padded [B, Tmax]
// layout (a frame only ever depends on earlier-or-equal frames of its own clip that exist for every clip length),
// the positional conv sees zeros past the clip's last frame, and the transformer runs on the packed valid frames.
// front_out != nullptr: stop after the positional convolution and write hidden_states[0] (the input of transformer
// layer 0: after encoder.layer_norm for the post-LN family, the positional-conv sum for the stable-layer-norm one).
static int hubert_forward_impl(const MerHubertModel* m, const float* wave, int B, int L, int normalize,
                               const int* lengths_host, void* workspace, long long workspace_bytes,
                               float* out_frames, float* out_utt, float* opt_hidden, void* stream_,
                               float* front_out = nullptr) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MER_REQUIRE(m && wave && workspace, "mer_hubert_forward: null operand");
  MER_REQUIRE(B > 0 && L > 0, "mer_hubert_forward: batch=%d n_samples=%d", B, L);
  MER_REQUIRE(m->readout == MER_HUBERT_READOUT_LAST4 || m->readout == MER_HUBERT_READOUT_LAST,
              "mer_hubert_forward: readout %d (MER_HUBERT_READOUT_LAST4 = 0 or MER_HUBERT_READOUT_LAST = 1)", m->readout);
  const bool last_only = m->readout == MER_HUBERT_READOUT_LAST;
  MER_REQUIRE(m->n_layers >= (last_only ? 1 : 4), "mer_hubert_forward: the %s readout needs >= %d layers (n_layers %d)",
              last_only ? "last-layer" : "last-four", last_only ? 1 : 4, m->n_layers);
  const int D = hub_dim(m), DFF = hub_ffn(m), HEADS = hub_heads(m);
  MER_REQUIRE((D == 768 || D == 1024) && HEADS * 64 == D && DFF % 128 == 0,
              "mer_hubert_forward: hidden %d / heads %d / ffn %d not supported", D, HEADS, DFF);
  MER_REQUIRE(!m->stable_layer_norm || m->pos_w_bd || m->n_pos_layers > 0,
              "mer_hubert_forward: the stable-layer-norm family needs pos_w_bd");
  const HubertPlan p = hubert_plan(B, L, D, DFF);
  MER_REQUIRE(p.T[6] > 0, "mer_hubert_forward: %d samples give no output frame", L);
  MER_REQUIRE(workspace_bytes >= p.total, "mer_hubert_forward: workspace %lld B < required %lld B",
              workspace_bytes, p.total);
  char* ws = static_cast<char*>(workspace);
  float* wave_n = reinterpret_cast<float*>(ws + p.off_wave);
  double* stats = reinterpret_cast<double*>(ws + p.off_stats);
  float* ping = reinterpret_cast<float*>(ws + p.off_ping);
  float* pong = reinterpret_cast<float*>(ws + p.off_pong);
  float* x = reinterpret_cast<float*>(ws + p.off_x);
  float* xs = reinterpret_cast<float*>(ws + p.off_xs);
  float* xn = reinterpret_cast<float*>(ws + p.off_xn);
  float* qkv = reinterpret_cast<float*>(ws + p.off_qkv);
  float* h = reinterpret_cast<float*>(ws + p.off_h);
  float* acc = reinterpret_cast<float*>(ws + p.off_acc);
  int* cu = reinterpret_cast<int*>(ws + p.off_cu);
  const int T = p.T[6];
  long long M = p.M;  // rows of the padded layout; becomes the packed frame count once a ragged batch is packed

  // ragged batch: per-clip extents, computed on the host and staged into the workspace
  const bool ragged = lengths_host != nullptr;
  int *d_len = nullptr, *d_t0 = nullptr, *d_tb = nullptr, *d_cu = nullptr;
  long long M_packed = 0;
  if (ragged) {
    MER_REQUIRE((m->pos_w_bd || m->n_pos_layers > 0) && !opt_hidden,
                "mer_hubert_forward_ragged: needs the GEMM positional conv; hidden states are not returned");
    std::vector<int> meta(4 * (size_t)B + 1);
    int* h_len = meta.data();
    int* h_t0 = h_len + B;
    int* h_tb = h_t0 + B;
    int* h_cu = h_tb + B;
    h_cu[0] = 0;
    for (int b = 0; b < B; ++b) {
      int t = lengths_host[b];
      MER_REQUIRE(t > 0 && t <= L, "mer_hubert_forward_ragged: clip %d has %d samples (row length %d)", b, t, L);
      h_len[b] = t;
      for (int i = 0; i < 7; ++i) {
        t = (t - kHubK[i]) / kHubS[i] + 1;
        if (i == 0) h_t0[b] = t;
      }
      MER_REQUIRE(t > 0, "mer_hubert_forward_ragged: clip %d (%d samples) gives no output frame", b, lengths_host[b]);
      h_tb[b] = t;
      h_cu[b + 1] = h_cu[b] + t;
    }
    M_packed = h_cu[B];
    d_len = reinterpret_cast<int*>(ws + p.off_meta);
    d_t0 = d_len + B;
    d_tb = d_t0 + B;
    d_cu = d_tb + B;
    // pageable source: the call returns once the data is staged, so `meta` may go out of scope afterwards
    MER_CUDA_CHECK(cudaMemcpyAsync(d_len, meta.data(), meta.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
  }

  // conv1 (and conv2) on fp16 operands when the model carries fp16 copies of their weights (group-norm family only):
  // conv0 / conv1 then write fp16 rows [clip][frame][512] -- same strides in elements as the split rows in 4-byte slots
  const bool f16_conv1 = !m->feat_norm_layer && m->conv_w_f16[0] != nullptr;
  const bool f16_conv2 = f16_conv1 && m->conv_w_f16[1] != nullptr;
  const float* wsrc = wave;
  if (normalize) {
    MER_TRY(mer_wave_normalize_launch(wave, wave_n, B, L, L, L, stream, d_len));
    wsrc = wave_n;
  }
  // conv0 + GroupNorm + GELU (or, layer-norm family: conv0 + bias + LayerNorm + GELU) -> ping [B, Tpad0, 512]
  if (m->feat_norm_layer) {
    MER_TRY(mer_hubert_conv0_ln_launch(wsrc, L, B, L, m->conv0_w, m->conv_b[0], m->conv_ln_g[0], m->conv_ln_b[0],
                                       ping, (long long)p.Tpad[0] * 512, stream));
  } else {
    MER_TRY(mer_hubert_conv0_launch(wsrc, L, B, L, m->conv0_w, m->gn_g, m->gn_b, stats, ping,
                                    (long long)p.Tpad[0] * 512, /*split_out=*/f16_conv1 ? 2 : 1, stream, d_t0));
  }
  // conv1..6 as implicit GEMMs over the time-major activations
  float* src = ping;
  float* dst = pong;
  for (int i = 1; i < 7; ++i) {
    MerGemmDesc g;
    memset(&g, 0, sizeof(g));
    const bool in16 = (i == 1 && f16_conv1) || (i == 2 && f16_conv2);  // this conv's operands are fp16
    const bool out16 = i == 1 && f16_conv2;                             // ... and so are the next one's
    g.A = src;
    g.W = in16 ? static_cast<const float*>(m->conv_w_f16[i - 1]) : m->conv_w[i - 1];
    g.rows_per_batch = p.T[i];
    g.a_rows_dim = p.Tpad[i - 1] / 2;
    g.batches = B;
    g.N = 512;
    g.K_inner = 512;
    g.taps = kHubK[i];
    g.P = 2;
    g.a_phase_stride = 512;
    g.a_row_stride = 1024;
    g.a_batch_stride = (long long)p.Tpad[i - 1] * 512;
    g.ep.out = dst;
    g.ep.out_bstride = (i == 6) ? p.T[6] : p.Tpad[i];  // conv6 output is packed [B*T, 512]
    g.ep.ld_out = 512;
    g.ep.split_off = 512;
    g.mode = in16 ? MER_GEMM_F16 : MER_GEMM_BF16X3;
    if (m->feat_norm_layer) {
      // conv + bias -> fp32; LayerNorm(512) + GELU in place -> split rows (conv6: fp32, it feeds another LayerNorm)
      g.ep.bias = m->conv_b[i];
      g.ep.flags = 0;
      MER_TRY(mer_gemm_launch(&g, stream));
      const long long rows = (i == 6) ? (long long)B * p.T[6] : (long long)B * p.Tpad[i];
      MER_TRY(mer_layernorm_launch(dst, m->conv_ln_g[i], m->conv_ln_b[i], i == 6 ? dst : nullptr,
                                   i == 6 ? nullptr : dst, nullptr, rows, 512, 1e-5f, MER_LN_GELU, stream));
    } else {
      g.ep.flags = MER_EPI_GELU | (i == 6 ? 0 : out16 ? MER_EPI_OUT_F16 : MER_EPI_SPLIT_BF16);  // conv6 feeds a LayerNorm: fp32
      if (in16) {  // timed as a class of its own (bench.py): not one of the ViT's linear layers
        const int prof = mer_prof_begin(MER_PROF_CONV_F16, 2.0 * (double)B * p.T[i] * 512.0 * 512.0 * kHubK[i], stream);
        mer_prof_pause(1);
        const int rc = mer_gemm_launch(&g, stream);
        mer_prof_pause(0);
        mer_prof_end(prof, stream);
        if (rc) return rc;
      } else {
        MER_TRY(mer_gemm_launch(&g, stream));
      }
    }
    float* tmp = src;
    src = dst;
    dst = tmp;
  }
  float* feat = src;  // [M, 512]
  // feature projection: LayerNorm(512) -> Linear 512->768  (x0 lands in the qkv buffer)
  MER_TRY(mer_layernorm_launch(feat, m->fp_ln_g, m->fp_ln_b, nullptr, feat, nullptr, M, 512,
                               m->ln_eps, 0, stream));
  float* x0 = qkv;
  MER_TRY(linear(MER_GEMM_BF16X3, feat, m->fp_w, m->fp_b, nullptr, x0, M, D, 512, 0, stream));
  // positional conv + GELU + residual -> xn
  MER_TRY(mer_iota_offsets_launch(cu, B, T, stream));
  if (m->n_pos_layers > 0) {
    // data2vec-audio: p_0 = x0;  p_{l+1} = GELU(LayerNorm_noaffine(conv_l(p_l) + b_l));  x1 = x0 + p_L.  Every conv is
    // the windowed block-diagonal fp16 GEMM of the classic positional conv with pos_taps taps and padding taps / 2.
    MER_REQUIRE(m->n_pos_layers <= 8 && (m->pos_taps & 1) && m->ln_ones && m->ln_zeros,
                "mer_hubert_forward: data2vec positional conv chain (%d layers, %d taps)", m->n_pos_layers, m->pos_taps);
    void* ph = h;  // fp16 copy of the current chain input (the FFN buffer is still unused)
    const int gch = D / 16;
    const int window = m->pos_window > 0 ? m->pos_window : 320;
    const float* cur = x0;
    for (int l = 0; l < m->n_pos_layers; ++l) {
      MER_REQUIRE(m->pos_layers_w[l] && m->pos_layers_b[l], "mer_hubert_forward: positional conv layer %d missing", l);
      MER_TRY(mer_cast_f16_launch(cur, ph, M * D, stream));
      if (ragged) MER_TRY(mer_zero_tail_rows_f16_launch(ph, d_tb, B, T, D, stream));
      MerGemmDesc g;
      memset(&g, 0, sizeof(g));
      g.A = static_cast<const float*>(ph);
      g.W = static_cast<const float*>(m->pos_layers_w[l]);
      g.rows_per_batch = T;
      g.a_rows_dim = T;
      g.batches = B;
      g.N = D;
      g.K_inner = window;
      g.taps = m->pos_taps;
      g.P = 1;
      g.a_phase_stride = D;
      g.a_row_stride = D;
      g.a_batch_stride = (long long)T * D;
      g.a_row0 = -(m->pos_taps / 2);
      g.a_cols = D;
      g.a_col_group = gch;
      g.force_block_n = 256;
      g.mode = MER_GEMM_F16;
      g.ep.bias = m->pos_layers_b[l];
      g.ep.out = xn;
      g.ep.out_bstride = T;
      g.ep.ld_out = D;
      MER_TRY(mer_gemm_launch(&g, stream));
      MER_TRY(mer_layernorm_launch(xn, m->ln_ones, m->ln_zeros, xn, nullptr, nullptr, M, D, 1e-5f, MER_LN_GELU, stream));
      cur = xn;
    }
    MER_TRY(mer_accumulate_launch(x0, xn, M * D, 0, stream));  // x1 = p_L + x0
  } else if (m->pos_w_bd) {
    // grouped conv (k = 128, 16 groups of 48 channels, zero padding 64, last frame dropped) as ONE fp16 GEMM
    // over windowed block-diagonal weights: output block j (256 columns) reads the 320-channel window that
    // starts at floor(256 j / 48) * 48; tap k reads frame t + k - 64 (rows outside the clip are zero).
    // 6.67x the algorithmic FLOPs, still ~2x faster than the mma.sync kernel.  x1 = x0 + GELU(conv + bias).
    void* x0h = h;  // fp16 copy of x0 in the (still unused) FFN buffer
    const int gch = D / 16;                                   // channels per group: 48 or 64
    const int window = m->pos_window > 0 ? m->pos_window : 320;
    const int prof = mer_prof_begin(MER_PROF_POSCONV, 2.0 * (double)M * D * gch * 128.0, stream);
    mer_prof_pause(1);
    int rc = mer_cast_f16_launch(x0, x0h, M * D, stream);
    if (rc == 0 && ragged) rc = mer_zero_tail_rows_f16_launch(x0h, d_tb, B, T, D, stream);  // conv padding = zeros
    if (rc == 0) {
      MerGemmDesc g;
      memset(&g, 0, sizeof(g));
      g.A = static_cast<const float*>(x0h);
      g.W = static_cast<const float*>(m->pos_w_bd);
      g.rows_per_batch = T;
      g.a_rows_dim = T;
      g.batches = B;
      g.N = D;
      g.K_inner = window;
      g.taps = 128;
      g.P = 1;
      g.a_phase_stride = D;
      g.a_row_stride = D;
      g.a_batch_stride = (long long)T * D;
      g.a_row0 = -64;
      g.a_cols = D;
      g.a_col_group = gch;
      g.force_block_n = 256;
      g.mode = MER_GEMM_F16;
      g.ep.bias = m->pos_b;
      g.ep.res = x0;
      g.ep.res_bstride = T;
      g.ep.out = xn;
      g.ep.out_bstride = T;
      g.ep.ld_out = D;
      g.ep.ld_res = D;
      g.ep.flags = MER_EPI_GELU;
      rc = mer_gemm_launch(&g, stream);
    }
    mer_prof_pause(0);
    mer_prof_end(prof, stream);
    if (rc) return rc;
  } else {
    MER_TRY(mer_posconv_launch(x0, m->pos_w, m->pos_b, cu, B, T, xn, stream));
  }
  if (ragged) {
    // padded [B, Tmax, D] -> packed [sum T_b, D]; from here on the batch is a varlen batch like BERT's
    MER_TRY(mer_pack_rows_launch(xn, d_cu, B, T, D, x, stream));
    M = M_packed;
    MER_CUDA_CHECK(cudaMemcpyAsync(xn, x, (size_t)M * D * 4, cudaMemcpyDeviceToDevice, stream));
    cu = d_cu;
  }
  if (front_out) {
    const float* h0 = xn;
    if (!m->stable_layer_norm) {
      MER_TRY(mer_layernorm_launch(xn, m->enc_ln_g, m->enc_ln_b, x, nullptr, nullptr, M, D, m->ln_eps, 0, stream));
      h0 = x;
    }
    MER_CUDA_CHECK(cudaMemcpyAsync(front_out, h0, (size_t)M * D * 4, cudaMemcpyDeviceToDevice, stream));
    return 0;
  }
  MerStackArgs a;
  memset(&a, 0, sizeof(a));
  a.eps = m->ln_eps;
  a.dim = D;
  a.ffn = DFF;
  a.heads = HEADS;
  a.tokens = M;
  a.cu_seqlens = cu;
  a.n_seq = B;
  a.max_seqlen = T;
  a.x = x;
  a.xs = xs;
  a.xn = xn;
  a.qkv = qkv;
  a.h = h;
  a.vt = reinterpret_cast<float*>(ws + p.off_vt);
  a.vt_ld = (M + 7) & ~7ll;
  a.hidden0_done = 1;
  a.long_rows = 1;
  const size_t hs_bytes = (size_t)M * D * 4;
  if (!m->stable_layer_norm) {
    // encoder.layer_norm -> x ; post-LN layers; readout = sum of the last four LayerNorm outputs
    // layers_f16 given: the 12 layers run on fp16 operands (the conv feature encoder above stays BF16X3: it has no
    // normalisation between its layers and is where the operand precision matters, scripts/precision_table.py)
    const bool f16 = m->layers_f16 != nullptr;
    MER_TRY(mer_layernorm_launch(xn, m->enc_ln_g, m->enc_ln_b, x, xs, nullptr, M, D, m->ln_eps,
                                 f16 ? MER_LN_SPLIT_F16 : 0, stream));
    if (opt_hidden) MER_CUDA_CHECK(cudaMemcpyAsync(opt_hidden, x, hs_bytes, cudaMemcpyDeviceToDevice, stream));
    a.layers = f16 ? m->layers_f16 : m->layers;
    a.n_layers = m->n_layers;
    a.pre_ln = 0;
    a.mode = f16 ? MER_GEMM_F16 : MER_GEMM_BF16X3;
    a.acc = acc;
    a.acc_last = last_only ? 1 : 4;  // hidden_states[-1] alone: the last layer's LayerNorm initialises acc
    a.opt_hidden = opt_hidden;
    MER_TRY(mer_run_stack(a, stream));
  } else {
    // HubertEncoderStableLayerNorm: the positional-conv sum is hidden state 0; pre-LN layers (BF16X3 like
    // the rest of the audio path, any sequence length); hidden states are the residual stream BEFORE each
    // layer, and encoder.layer_norm of the
    // last one closes the tuple: readout = x_{L-4} + x_{L-3} + x_{L-2} + LayerNorm(x_{L-1})
    // (x_l = stream after layer l).
    MER_CUDA_CHECK(cudaMemcpyAsync(x, xn, hs_bytes, cudaMemcpyDeviceToDevice, stream));
    if (opt_hidden) MER_CUDA_CHECK(cudaMemcpyAsync(opt_hidden, x, hs_bytes, cudaMemcpyDeviceToDevice, stream));
    a.pre_ln = 1;
    const bool f16 = m->layers_f16 != nullptr && mer_attention_f16_supported(T);
    a.mode = f16 ? MER_GEMM_F16 : MER_GEMM_BF16X3;
    const MerLayerWeights* layers = f16 ? m->layers_f16 : m->layers;
    const int L0 = m->n_layers - 4;  // layers before the readout window
    int done = 0;
    auto run = [&](int n) -> int {
      a.layers = layers + done;
      a.n_layers = n;
      a.opt_hidden = opt_hidden ? opt_hidden + (size_t)done * M * D : nullptr;
      const int rc = n > 0 ? mer_run_stack(a, stream) : 0;
      done += n;
      return rc;
    };
    if (last_only) {
      // hidden_states[-1] alone = encoder.layer_norm of the last layer's output
      MER_TRY(run(m->n_layers));
      float* last = opt_hidden ? opt_hidden + (size_t)m->n_layers * M * D : xn;
      MER_TRY(mer_layernorm_launch(x, m->enc_ln_g, m->enc_ln_b, last, nullptr, acc, M, D, m->ln_eps, MER_LN_ACC_INIT,
                                   stream));
    } else {
      MER_TRY(run(L0 + 1));                                      // x = x_{L-4}
      MER_TRY(mer_accumulate_launch(x, acc, M * D, 1, stream));
      for (int k = 0; k < 2; ++k) {
        MER_TRY(run(1));                                         // x_{L-3}, x_{L-2}
        MER_TRY(mer_accumulate_launch(x, acc, M * D, 0, stream));
      }
      MER_TRY(run(1));                                           // x_{L-1}
      float* last = opt_hidden ? opt_hidden + (size_t)m->n_layers * M * D : xn;
      MER_TRY(mer_layernorm_launch(x, m->enc_ln_g, m->enc_ln_b, last, nullptr, acc, M, D, m->ln_eps,
                                   MER_LN_ACC_ADD, stream));
    }
  }
  if (out_frames)
    MER_CUDA_CHECK(cudaMemcpyAsync(out_frames, acc, hs_bytes, cudaMemcpyDeviceToDevice, stream));
  if (out_utt)
    MER_TRY(mer_segment_reduce_launch(acc, cu, cu + 1, B, D, MER_SEG_MEAN, out_utt, stream));
  return 0;
}

int mer_hubert_forward(const MerHubertModel* m, const float* wave, int B, int L, int normalize,
                       void* workspace, long long workspace_bytes, float* out_frames, float* out_utt,
                       float* opt_hidden, void* stream) {
  return hubert_forward_impl(m, wave, B, L, normalize, nullptr, workspace, workspace_bytes, out_frames, out_utt,
                             opt_hidden, stream);
}

int mer_hubert_frontend(const MerHubertModel* m, const float* wave, int B, int L, int normalize, void* workspace,
                        long long workspace_bytes, float* out_hidden0, void* stream) {
  MER_REQUIRE(out_hidden0, "mer_hubert_frontend: null output");
  return hubert_forward_impl(m, wave, B, L, normalize, nullptr, workspace, workspace_bytes, nullptr, nullptr, nullptr,
                             stream, out_hidden0);
}

int mer_hubert_forward_ragged(const MerHubertModel* m, const float* wave, const int* lengths_host, int B, int L,
                              int normalize, void* workspace, long long workspace_bytes, float* out_frames,
                              float* out_utt, void* stream) {
  MER_REQUIRE(lengths_host, "mer_hubert_forward_ragged: null lengths");
  return hubert_forward_impl(m, wave, B, L, normalize, lengths_host, workspace, workspace_bytes, out_frames, out_utt,
                             nullptr, stream);
}

// ------------------------------------------------------------------------------------------------
// BERT / RoBERTa
// ------------------------------------------------------------------------------------------------
static long long bert_ws(long long M, int D, int DFF) {
  return (M * (D + D + D + 3ll * D + DFF + D) + (long long)D * ((M + 7) & ~7ll)) * 4 + 4096;
}
static int bert_dim(const MerBertModel* m) { return m->hidden > 0 ? m->hidden : ::D; }
static int bert_ffn(const MerBertModel* m) { return m->ffn > 0 ? m->ffn : ::DFF; }

long long mer_bert_workspace_bytes(int tokens, int n_seq) {
  (void)n_seq;
  return bert_ws(tokens, ::D, ::DFF);
}

long long mer_bert_model_workspace_bytes(const MerBertModel* m, int tokens, int n_seq) {
  (void)n_seq;
  if (!m) return -1;
  return bert_ws(tokens, bert_dim(m), bert_ffn(m));
}

// proj == NULL: BERT / RoBERTa / ELECTRA with embedding_size == hidden_size; otherwise ELECTRA's factorised embedding
// (LayerNorm at width E, then the E -> H projection writes hidden state 0)
static int bert_forward_impl(const MerBertModel* m, const MerBertEmbedProjection* proj, const int32_t* ids,
                             const int32_t* pos_ids, const int32_t* cu_seqlens, int n_seq, int tokens, int max_seqlen,
                             const int32_t* seg_begins, const int32_t* seg_ends, void* workspace,
                             long long workspace_bytes, float* out_tokens, float* out_utt, float* opt_hidden,
                             cudaStream_t stream) {
  MER_REQUIRE(m && ids && pos_ids && cu_seqlens && workspace, "mer_bert_forward: null operand");
  MER_REQUIRE(n_seq > 0 && tokens > 0 && max_seqlen > 0, "mer_bert_forward: empty batch");
  MER_REQUIRE(m->n_layers >= 4, "mer_bert_forward: the last-four readout needs >= 4 layers");
  // model dims: zero-initialised fields = the base models (768 / 12 heads / 3072); -large: 1024 / 16 / 4096;
  // ELECTRA-small / LERT-small: 256 / 4 / 1024
  const int D = bert_dim(m), DFF = bert_ffn(m), HEADS = m->heads > 0 ? m->heads : ::HEADS, DQKV = 3 * D;
  MER_REQUIRE((D == 768 || D == 1024 || D == 256) && HEADS * 64 == D && DFF % 128 == 0,
              "mer_bert_forward: hidden %d / heads %d / ffn %d not supported", D, HEADS, DFF);
  MER_REQUIRE(workspace_bytes >= bert_ws(tokens, D, DFF), "mer_bert_forward: workspace %lld B < required %lld B",
              workspace_bytes, bert_ws(tokens, D, DFF));
  const bool f16 = m->layers_f16 != nullptr;
  const long long M = tokens;
  float* x = static_cast<float*>(workspace);
  float* xs = x + M * D;
  float* xn = xs + M * D;
  float* qkv = xn + M * D;
  float* h = qkv + M * DQKV;
  float* acc = h + M * DFF;
  float* vt = acc + M * D;
  if (proj) {
    const int E = proj->emb_dim;
    MER_REQUIRE((E == 128 || E == 256) && E != D, "mer_bert_forward_projected: embedding size %d (128 or 256, != hidden %d)",
                E, D);
    // the E-wide LayerNorm output and its GEMM operand live in the FFN buffer, idle before layer 1
    MER_REQUIRE(2 * E <= DFF, "mer_bert_forward_projected: embedding size %d needs 2 x %d <= ffn %d", E, E, DFF);
    MER_REQUIRE(proj->word_emb && proj->pos_emb && proj->type_emb0 && proj->emb_ln_g && proj->emb_ln_b && proj->proj_b &&
                    (f16 ? proj->proj_w_f16 != nullptr : proj->proj_w != nullptr),
                "mer_bert_forward_projected: null table or weight (the %s projection)", f16 ? "fp16" : "split bf16");
    float* e32 = h;           // [M, E] fp32 LayerNorm_E output
    float* eop = h + M * E;   // [M, E] its GEMM operand: split bf16 rows (E 4-byte slots) or fp16 rows
    MER_TRY(mer_bert_embed_launch(ids, pos_ids, proj->word_emb, proj->pos_emb, proj->type_emb0, proj->emb_ln_g,
                                  proj->emb_ln_b, m->ln_eps, tokens, e32, f16 ? nullptr : eop, stream, E));
    if (f16) MER_TRY(mer_cast_f16_launch(e32, eop, M * E, stream));
    const float* pw = f16 ? static_cast<const float*>(proj->proj_w_f16) : proj->proj_w;
    MER_TRY(linear(f16 ? MER_GEMM_F16 : MER_GEMM_BF16X3, eop, pw, proj->proj_b, nullptr, x, M, D, E, 0, stream));
    // the stack's operand copy of hidden state 0
    if (f16) MER_TRY(mer_cast_f16_launch(x, xs, M * D, stream));
    else MER_TRY(mer_split_bf16(x, xs, M, D, stream));
  } else {
    MER_REQUIRE(m->word_emb && m->pos_emb && m->type_emb0 && m->emb_ln_g && m->emb_ln_b,
                "mer_bert_forward: null embedding table");
    MER_TRY(mer_bert_embed_launch(ids, pos_ids, m->word_emb, m->pos_emb, m->type_emb0, m->emb_ln_g,
                                  m->emb_ln_b, m->ln_eps, tokens, x, xs, stream, D));
    if (f16) MER_TRY(mer_cast_f16_launch(x, xs, M * D, stream));  // the embedding LayerNorm's fp16 copy (operand)
  }
  if (opt_hidden)
    MER_CUDA_CHECK(cudaMemcpyAsync(opt_hidden, x, (size_t)M * D * 4, cudaMemcpyDeviceToDevice, stream));
  MerStackArgs a;
  memset(&a, 0, sizeof(a));
  a.layers = f16 ? m->layers_f16 : m->layers;
  a.n_layers = m->n_layers;
  a.pre_ln = 0;
  a.dim = D;
  a.ffn = DFF;
  a.heads = HEADS;
  a.mode = f16 ? MER_GEMM_F16 : MER_GEMM_BF16X3;
  a.eps = m->ln_eps;
  a.tokens = M;
  a.cu_seqlens = cu_seqlens;
  a.n_seq = n_seq;
  a.max_seqlen = max_seqlen;
  a.x = x;
  a.xs = xs;
  a.xn = xn;
  a.qkv = qkv;
  a.h = h;
  a.acc = acc;
  a.acc_last = 4;
  a.vt = vt;
  a.vt_ld = (M + 7) & ~7ll;  // fp32 or fp16 V^T rows start on 16-byte boundaries
  a.opt_hidden = opt_hidden;
  a.hidden0_done = 1;
  MER_TRY(mer_run_stack(a, stream));
  if (out_tokens)
    MER_CUDA_CHECK(cudaMemcpyAsync(out_tokens, acc, (size_t)M * D * 4, cudaMemcpyDeviceToDevice, stream));
  if (out_utt && seg_begins && seg_ends)
    MER_TRY(mer_segment_reduce_launch(acc, seg_begins, seg_ends, n_seq, D, MER_SEG_MEAN, out_utt, stream));
  return 0;
}

int mer_bert_forward(const MerBertModel* m, const int32_t* ids, const int32_t* pos_ids,
                     const int32_t* cu_seqlens, int n_seq, int tokens, int max_seqlen,
                     const int32_t* seg_begins, const int32_t* seg_ends, void* workspace,
                     long long workspace_bytes, float* out_tokens, float* out_utt, float* opt_hidden,
                     void* stream) {
  return bert_forward_impl(m, nullptr, ids, pos_ids, cu_seqlens, n_seq, tokens, max_seqlen, seg_begins, seg_ends,
                           workspace, workspace_bytes, out_tokens, out_utt, opt_hidden, static_cast<cudaStream_t>(stream));
}

int mer_bert_forward_projected(const MerBertModel* m, const MerBertEmbedProjection* proj, const int32_t* ids,
                               const int32_t* pos_ids, const int32_t* cu_seqlens, int n_seq, int tokens, int max_seqlen,
                               const int32_t* seg_begins, const int32_t* seg_ends, void* workspace,
                               long long workspace_bytes, float* out_tokens, float* out_utt, float* opt_hidden,
                               void* stream) {
  return bert_forward_impl(m, proj, ids, pos_ids, cu_seqlens, n_seq, tokens, max_seqlen, seg_begins, seg_ends,
                           workspace, workspace_bytes, out_tokens, out_utt, opt_hidden, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
